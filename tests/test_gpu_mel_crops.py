"""Mel crop batches: Corpus.mel_crops and clx_batch_create_mel_crops (-m gpu).

Every batch is compared with tests/spec_mel.py (float64) applied to the float32 output of the equivalent CropBatch (the
resampled one with sample_rate) given the same requests, within spec_mel.check's tolerance; status, lengths and the
error word must be that batch's.  Host corpora and attached images must give a device corpus's features bit for bit.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from tests import spec_mel as S
from tests import spec_resample as SR
from tests.test_gpu_corpus import c4ch_config, damaged_index, flac_of
from tests.test_gpu_resampled_crops import cfg_at, mixed_files, mono
from tests.test_gpu_shared_corpus import image_path

gpu = pytest.mark.gpu

GRID = [  # n_fft, win_length, hop, center, n_mels, f_min, f_max, mel_scale, norm, L
    (8, 8, 1, True, 1, 0.0, None, "htk", None, 5),
    (8, 5, 9, False, 1, 0.0, None, "slaney", "slaney", 100),
    (30, 27, 7, True, 1, 100.0, None, "htk", "slaney", 16),
    (320, 300, 160, True, 80, 0.0, 7600.0, "slaney", "slaney", 1003),
    (400, 301, 400, False, 80, 20.0, None, "htk", None, 4099),
    (400, 400, 160, True, 128, 0.0, None, "htk", None, 201),
    (512, 511, 777, True, 128, 0.0, None, "slaney", None, 3001),
    (2048, 1024, 512, False, 80, 30.0, 7000.0, "htk", "slaney", 5000),
    (4096, 4096, 4096, True, 128, 0.0, None, "htk", None, 9000),
]
WORST = [0.0]  # the largest error-to-bound ratio seen


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


_files = {}


def single_rate_files():
    """Files at 44.1 kHz of 1, 2 and 4 channels (C = 4)."""
    if "single" not in _files:
        _files["single"] = [flac_of(cfg_at(synth.workload_config("c2", 9), 44100)),
                            flac_of(cfg_at(c4ch_config(), 44100)), flac_of(cfg_at(mono(5, 4096, 31), 44100))]
    return _files["single"]


def mel_args(n_fft, win, hop, center, n_mels, f_min, f_max, scale, norm, log_floor=None):
    return dict(n_fft=n_fft, win_length=win, hop_length=hop, center=center, n_mels=n_mels, f_min=f_min, f_max=f_max,
                mel_scale=scale, norm=norm, log_floor=log_floor)


def reference(mb, x, rows=None):
    """spec_mel of the crop output x [B, C, L] with the batch's own window and filterbank: (ref, power bound)."""
    p = mb.params
    center = bool(p.flags & cb.MEL_CENTER)
    x = x if rows is None else x[rows]
    log_floor = float(p.log_floor) if p.flags & cb.MEL_LOG else None
    ref = S.mel(x, p.n_fft, p.hop_length, mb.window, mb.fbank, center, log_floor)
    return ref, S.bound(x, p.n_fft, p.hop_length, mb.window, mb.fbank, center), log_floor


def check_against_crops(mb, crops, files, offsets, rows=None):
    """One call of the mel batch and of its equivalent crop batch with the same requests; returns the features."""
    import torch
    x, lengths = crops(files, offsets, check=False)
    x = x.cpu().numpy()
    feats, ml = mb(files, offsets, check=False)
    assert feats.shape == (mb.batch, mb.channels, mb.n_mels, mb.n_frames) and feats.dtype == torch.float32
    assert torch.equal(ml, lengths) and torch.equal(mb.status, crops.status) and torch.equal(mb._error, crops._error)
    ref, delta, log_floor = reference(mb, x, rows)
    dev = feats.cpu().numpy()
    WORST[0] = max(WORST[0], S.check(dev if rows is None else dev[rows], ref, delta, log_floor))
    return dev


def edge_requests(idx, L, R=None):
    files, offsets = [], []
    for fi, f in enumerate(idx.files):
        N = f.length if R is None else SR.out_len(f.length, f.info.sample_rate, R)
        for o in sorted({0, 1, N // 3, max(0, N - L), max(0, N - L // 2), N - 1, N}):
            files.append(fi)
            offsets.append(o)
    return files, offsets


# --------------------------------------------------------------------------- 1. against the float64 reference

@gpu
def test_plain_crops_every_path(ctx):
    """A single-rate corpus, every decode path: power and log features of edge crops."""
    import torch
    idx = cb.index(single_rate_files())
    corpus = cb.Corpus(idx, ctx)
    L = 4000
    files, offsets = edge_requests(idx, L)
    crops = corpus.crops(len(files), L, dtype=torch.float32)
    for log_floor in (None, 1e-10):
        mb = corpus.mel_crops(len(files), L, n_fft=400, hop_length=160, n_mels=80, log_floor=log_floor)
        assert mb.channels == 4 and mb.n_frames == 1 + L // 160
        check_against_crops(mb, crops, files, offsets)


@gpu
@pytest.mark.parametrize("g", range(len(GRID)))
def test_resampled_crops_grid(rctx, g):
    """The mixed-rate corpus at 16 kHz over the parameter grid: n_fft 8 to 4096, windows shorter than n_fft by odd
    and even gaps, hops below, at and above n_fft, both center modes, L = n_fft / 2 + 1 and hops that do not divide L."""
    import torch
    *args, L = GRID[g]
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    files, offsets = edge_requests(idx, L, 16000)
    crops = corpus.crops(len(files), L, sample_rate=16000)
    for log_floor in (None, 1e-6):
        mb = corpus.mel_crops(len(files), L, 16000, **mel_args(*args, log_floor=log_floor))
        check_against_crops(mb, crops, files, offsets)
    if args[3]:  # the shortest row reflect padding allows
        n = args[0] // 2 + 1
        mb = corpus.mel_crops(len(files), n, 16000, **mel_args(*args))
        check_against_crops(mb, corpus.crops(len(files), n, sample_rate=16000), files, offsets)
    del crops
    gc.collect()
    assert WORST[0] <= 1.0
    print(f"worst error / bound so far: {WORST[0]:.3g}")


@gpu
@pytest.mark.parametrize("whisper", [False, True])
def test_against_torchaudio(rctx, whisper):
    """torchaudio.transforms.MelSpectrogram on the GPU, on the crop output: its defaults, and Whisper's front end (400 /
    160 / 128 mels, Slaney scale and norm), within the same bound (with torchaudio's own float32 filterbank)."""
    torch = pytest.importorskip("torch")
    T = pytest.importorskip("torchaudio")
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    L = 16000
    files, offsets = edge_requests(idx, L, 16000)
    crops = corpus.crops(len(files), L, sample_rate=16000)
    kw = dict(n_fft=400, hop_length=160, n_mels=128, norm="slaney", mel_scale="slaney") if whisper else {}
    mb = corpus.mel_crops(len(files), L, 16000, **kw)
    x, _ = crops(files, offsets, check=False)
    ref = T.transforms.MelSpectrogram(16000, **kw).cuda()(x).cpu().double().numpy()
    fb_ta = T.functional.melscale_fbanks(201, 0.0, 8000.0, 128, 16000, kw.get("norm"), kw.get("mel_scale", "htk"))
    feats, _ = mb(files, offsets, check=False)
    p, x = mb.params, x.cpu().numpy()
    # each side's bound, plus what the difference of torchaudio's float32 filterbank from ours can make
    pw = S.power(x, p.n_fft, p.hop_length, mb.window, True)
    fb_diff = np.abs(fb_ta.double().numpy() - mb.fbank.astype(np.float64))
    tol = 2 * S.bound(x, p.n_fft, p.hop_length, mb.window, mb.fbank, True) + np.swapaxes(pw @ fb_diff, -1, -2)
    err = np.abs(feats.cpu().double().numpy() - ref)
    assert feats.shape == ref.shape
    assert (err <= tol).all(), (err / np.maximum(tol, 1e-30)).max()


# --------------------------------------------------------------------------- 2. invalid requests, damaged files

@gpu
def test_invalid_requests(rctx):
    """Features exactly 0, or exactly ln(log_floor) rounded to float32, after a call that filled them."""
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    L, R = 3000, 16000
    files, offsets = edge_requests(idx, L, R)
    bad = {1: (len(idx), 0), 4: (0, -1), 6: (2, SR.out_len(idx[2].length, 8000, R) + 1), 9: ((1 << 32) + 1, 0)}
    for log_floor in (None, 1e-10, 3.5):
        mb = corpus.mel_crops(len(files), L, R, n_mels=64, log_floor=log_floor)
        mb(files, offsets, check=False)
        f2, o2 = list(files), list(offsets)
        for b, (f, o) in bad.items():
            f2[b], o2[b] = f, o
        feats, lengths = mb(f2, o2, check=False)
        want = 0.0 if log_floor is None else float(np.float32(np.log(log_floor)))
        feats, status = feats.cpu().numpy(), mb.status.cpu().numpy()
        for b in bad:
            assert status[b] == 90 and lengths[b] == 0
            assert (feats[b] == np.float32(want)).all(), (b, log_floor)
        with pytest.raises(ValueError, match="crop 1: file index"):
            mb(f2, o2)


@gpu
def test_damaged_files(rctx, golden):
    """Status, lengths and the error word are the resampled crop batch's; check=True raises what it raises."""
    import torch
    idx = damaged_index(golden)
    corpus = cb.Corpus(idx, rctx)
    R, L = 16000, 3000
    files, offsets = edge_requests(idx, L, R)
    crops = corpus.crops(len(files), L, sample_rate=R)
    mb = corpus.mel_crops(len(files), L, R, n_mels=40)
    crops(files, offsets, check=False)
    mb(files, offsets, check=False)
    assert torch.equal(mb.status, crops.status) and torch.equal(mb.lengths, crops.lengths)
    assert torch.equal(mb._error, crops._error) and mb.status.any()
    with pytest.raises(cb.Error) as ea:
        crops(files, offsets)
    with pytest.raises(cb.Error) as eb:
        mb(files, offsets)
    assert str(ea.value) == str(eb.value)


# --------------------------------------------------------------------------- 3. determinism, requests on the device

@gpu
def test_bit_identical_calls(rctx):
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    L, R = 8000, 16000
    files, offsets = edge_requests(idx, L, R)
    mb = corpus.mel_crops(len(files), L, R, log_floor=1e-10)
    a = mb(files, offsets)[0].clone()
    assert torch.equal(mb(files, offsets)[0], a)
    mb(files[::-1], offsets[::-1])  # a different call in between
    b = mb(files, offsets)[0].clone()
    fresh = corpus.mel_crops(len(files), L, R, log_floor=1e-10)
    assert torch.equal(b.view(torch.int32), a.view(torch.int32))
    assert torch.equal(fresh(files, offsets)[0].view(torch.int32), a.view(torch.int32))


@gpu
def test_device_drawn_requests_without_sync(rctx):
    """Requests drawn on the GPU, check=False under sync debug mode "error", two batches interleaved."""
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    nt = torch.tensor([SR.out_len(f.length, f.info.sample_rate, R) for f in idx.files], device="cuda")
    a = corpus.mel_crops(12, 20000, R, log_floor=1e-10)
    b = corpus.mel_crops(9, 777, R, n_fft=512, hop_length=100, n_mels=40)
    gen = torch.Generator(device="cuda").manual_seed(7)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            for batch in (a, b):
                fi = torch.randint(0, len(idx), (batch.batch,), device="cuda", generator=gen)
                off = torch.minimum((torch.rand(batch.batch, device="cuda", generator=gen) * (nt[fi] + 1)).long(), nt[fi])
                batch(fi, off, check=False)
                draws.append((batch, fi, off, batch.out.clone(), batch.status.clone()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for batch, fi, off, feats, status in draws:
        assert not status.any()
        crops = corpus.crops(batch.batch, batch.num_frames, sample_rate=R)
        x, _ = crops(fi, off)
        ref, delta, log_floor = reference(batch, x.cpu().numpy())
        S.check(feats.cpu().numpy(), ref, delta, log_floor)


# --------------------------------------------------------------------------- 4. corpora, launches

@gpu
def test_host_and_attached_corpora(rctx):
    import torch
    srcs = mixed_files()
    idx = cb.index(srcs)
    L, R = 5000, 16000
    files, offsets = edge_requests(idx, L, R)
    dev = cb.Corpus(idx, rctx).mel_crops(len(files), L, R, log_floor=1e-10)
    want = dev(files, offsets)[0].clone()
    with image_path() as path:
        shared = cb.Corpus.share(idx, path, rctx)
        attached = cb.Corpus.attach(path, rctx)
    for c in (cb.Corpus(idx, rctx, memory="host"), shared, attached):
        mb = c.mel_crops(len(files), L, R, log_floor=1e-10)
        got = mb(files, offsets)[0]
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), c.memory
        del mb, got  # (the views keep the batch, and the batch its corpus, alive)
    gc.collect()
    attached.close()
    shared.close()


@gpu
def test_launch_counts(rctx):
    """A call launches what its crop batch launches, plus mel_kernel."""
    import torch
    idx = cb.index(mixed_files())
    one = cb.index(single_rate_files())

    def per_call(batch, *args):
        batch(*args, check=False)
        n0 = rctx.launch_count
        batch(*args, check=False)
        return rctx.launch_count - n0

    B, L = 7, 5000
    for c in (cb.Corpus(idx, rctx), cb.Corpus(idx, rctx, memory="host")):
        req = (list(range(B)), [0] * B)
        assert per_call(c.mel_crops(B, L, 16000), *req) == per_call(c.crops(B, L, sample_rate=16000), *req) + 1
    for c in (cb.Corpus(one, rctx), cb.Corpus(one, rctx, memory="host")):
        req = ([0, 1, 2] * 2, [0] * 6)
        assert per_call(c.mel_crops(6, L), *req) == per_call(c.crops(6, L, dtype=torch.float32), *req) + 1


# --------------------------------------------------------------------------- 5. refusals

@gpu
def test_refusals(rctx):
    import torch
    Lb = rctx._L
    idx = cb.index(mixed_files()[:3])
    corpus = cb.Corpus(idx, rctx)
    rates = np.array([f.info.sample_rate for f in idx.files], np.uint32)
    good = dict(n_fft=400, win_length=400, hop_length=160, n_mels=80, flags=cb.MEL_CENTER, log_floor=0.0)
    b = C.c_void_p()

    def create(n_crops=4, L=1000, R=16000, window=True, fbank=True, params=True, rates_=rates, n_files=3, **kw):
        p = {**good, **kw}
        mp = cb._lib.MelParams(p["n_fft"], p["win_length"], p["hop_length"], p["n_mels"], p["flags"], p["log_floor"])
        w = np.ones(max(1, p["win_length"]), np.float32)
        fb = np.ones((p["n_fft"] // 2 + 1, max(1, p["n_mels"])), np.float32)
        if isinstance(window, np.ndarray):
            w = window
        if isinstance(fbank, np.ndarray):
            fb = fbank
        rc = Lb.clx_batch_create_mel_crops(rctx._h, corpus._h, None if rates_ is None else rates_.ctypes.data, n_files,
                                           n_crops, L, R, C.byref(mp) if params else None,
                                           w.ctypes.data if window is not None else None,
                                           fb.ctypes.data if fbank is not None else None, C.byref(b))
        return rc

    assert create() == 0
    assert Lb.clx_batch_crop_requests(b) and Lb.clx_batch_packed_requests(b) is None
    Lb.clx_batch_destroy(rctx._h, b)
    assert create(n_fft=4096, win_length=1, hop_length=1, n_mels=512, L=2049, flags=3, log_floor=1e-30) == 0
    Lb.clx_batch_destroy(rctx._h, b)
    assert create(n_fft=8, win_length=8, n_mels=1, L=8, flags=0, R=0, rates_=None) == 0  # plain crops, no rates
    Lb.clx_batch_destroy(rctx._h, b)
    nan_w, nan_fb = np.ones(400, np.float32), np.ones((201, 80), np.float32)
    nan_w[7], nan_fb[3, 5] = np.nan, np.inf
    for kw in (dict(n_fft=402), dict(n_fft=401), dict(n_fft=6, win_length=6), dict(n_fft=4100, win_length=400),
               dict(n_fft=8192, win_length=400), dict(n_fft=14 * 2, win_length=20), dict(win_length=0),
               dict(win_length=401), dict(hop_length=0), dict(n_mels=0), dict(n_mels=513), dict(flags=4),
               dict(flags=3, log_floor=0.0), dict(flags=3, log_floor=-1.0), dict(flags=3, log_floor=float("inf")),
               dict(flags=3, log_floor=float("nan")), dict(log_floor=1e-10), dict(L=200), dict(L=399, flags=0),
               dict(params=False), dict(window=None), dict(fbank=None), dict(window=nan_w), dict(fbank=nan_fb),
               dict(n_crops=0), dict(n_crops=1 << 30), dict(L=0), dict(L=1 << 62), dict(R=655351),
               dict(rates_=None), dict(n_files=2), dict(n_crops=1 << 28, L=1 << 33)):
        assert create(**kw) == 90, kw
        assert not b.value
    for kw in (dict(L=201), dict(L=400, flags=0)):  # the shortest rows
        assert create(**kw) == 0, kw
        Lb.clx_batch_destroy(rctx._h, b)
    mixed = cb.Corpus(cb.index(mixed_files()), rctx)
    with pytest.raises(ValueError, match="sample rates"):
        mixed.mel_crops(4, 1000)
    with pytest.raises(cb.Error):
        mixed.mel_crops(4, 200, 16000)
    with pytest.raises(ValueError):
        mixed.mel_crops(4, 1000, 16000, mel_scale="kaldi")
    batch = mixed.mel_crops(2, 1000, 16000)
    with pytest.raises(cb.Error):
        mixed.close()
    del batch
    gc.collect()
    mixed.close()


# --------------------------------------------------------------------------- 6. the workload

@gpu
def test_workload_256_crops_of_10s(rctx):
    """256 stereo crops of 10 s at 16 kHz from 44.1 / 48 kHz files, n_fft 400, hop 160, 128 mels, log floor 1e-10,
    once; eight crops checked against the reference."""
    import torch
    rng = np.random.default_rng(1)
    srcs = []
    for i in range(8):
        cfg = synth.workload_config("c2", int(rng.integers(216, 431)), seed=100 + i)  # 20 to 40 s of 4096-sample frames
        srcs.append(flac_of(cfg_at(cfg, 44100 if i % 2 else 48000)))
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, rctx)
    R, L, B = 16000, 160000, 256
    mb = corpus.mel_crops(B, L, R, n_fft=400, hop_length=160, n_mels=128, log_floor=1e-10)
    crops = corpus.crops(B, L, sample_rate=R)
    files = rng.integers(0, len(idx), B)
    offsets = [int(rng.integers(0, max(1, SR.out_len(idx[f].length, idx[f].info.sample_rate, R) - L // 2)))
               for f in files]
    assert mb.out.shape == (B, 2, 128, 1001)
    check_against_crops(mb, crops, files, offsets, rows=[0, 1, 77, 128, 200, 253, 254, 255])
