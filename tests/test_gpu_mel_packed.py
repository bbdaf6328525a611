"""Mel packed batches: Corpus.mel_packed and clx_batch_create_mel_packed (-m gpu).

Every call is compared with the equivalent float32 PackedBatch (the resampled one with sample_rate) given the same
requests: excerpt b's frames against tests/spec_mel.py (float64) of its slice out[:, s_b : s_b + n_b], within
spec_mel.check's tolerance; frame counts and starts against the layout rule; every other element of the features
exactly 0; status, lengths and the error word the packed batch's.  An excerpt inside its file must give a MelCropBatch's
features bit for bit, and host corpora and attached images a device corpus's.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import claxon_b200 as cb
from tests import spec_mel as S
from tests import spec_resample as SR
from tests.test_gpu_mel_crops import GRID, mel_args, single_rate_files
from tests.test_gpu_resampled_crops import mixed_files
from tests.test_gpu_resampled_packed import r4
from tests.test_gpu_shared_corpus import image_path

gpu = pytest.mark.gpu
WORST = [0.0]  # the largest error-to-bound ratio seen


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


def n_frames(n, n_fft, hop, center):
    if n <= n_fft // 2 if center else n < n_fft:
        return 0
    return S.n_frames(n, n_fft, hop, center)


def lengths_at(idx, R=None):
    return [f.length if R is None else SR.out_len(f.length, f.info.sample_rate, R) for f in idx.files]


def check_call(mb, pk, files, offsets=None, lengths=None):
    """One call of the mel packed batch and of its packed batch `pk`; returns (features, starts, frames) on the host."""
    import torch
    x, s, n = pk(files, offsets, lengths, check=False)
    feats, starts, frames, ml = mb(files, offsets, lengths, check=False)
    assert feats.shape == (mb.channels, mb.n_mels, mb.stride) and feats.dtype == torch.float32
    assert torch.equal(ml, n) and torch.equal(mb.status, pk.status) and torch.equal(mb._error, pk._error)
    p = mb.params
    center = bool(p.flags & cb.MEL_CENTER)
    log_floor = float(p.log_floor) if p.flags & cb.MEL_LOG else None
    nn = n.cpu().numpy()
    want_f = [n_frames(int(v), p.n_fft, p.hop_length, center) for v in nn]
    want_s = np.concatenate([[0], np.cumsum([r4(f) for f in want_f])])[:-1].tolist() if want_f else []
    starts, frames = starts.cpu().numpy(), frames.cpu().numpy()
    assert frames.tolist() == want_f and starts.tolist() == want_s
    dev, x, s = feats.cpu().numpy(), x.cpu().numpy(), s.cpu().numpy()
    covered = np.zeros(dev.shape, dtype=bool)
    for b, F in enumerate(want_f):
        if not F:
            continue
        seg = x[:, s[b]:s[b] + nn[b]]
        ref = S.mel(seg, p.n_fft, p.hop_length, mb.window, mb.fbank, center, log_floor)
        delta = S.bound(seg, p.n_fft, p.hop_length, mb.window, mb.fbank, center)
        WORST[0] = max(WORST[0], S.check(dev[:, :, starts[b]:starts[b] + F], ref, delta, log_floor))
        covered[:, :, starts[b]:starts[b] + F] = True
    stray = np.nonzero(dev.view(np.int32) * ~covered)
    assert stray[0].size == 0, ("elements without a frame not 0", stray[2][:4])
    return dev, starts, frames


def requests(idx, L_of, rng, R=None, n=3):
    """Per file: the whole file, n random excerpts of L_of(rng) samples, and its last 77 samples."""
    files, offsets, lengths = [], [], []
    for fi, N in enumerate(lengths_at(idx, R)):
        files.append(fi), offsets.append(0), lengths.append(-1)
        for _ in range(n):
            L = L_of(rng)
            files.append(fi), offsets.append(int(rng.integers(0, N + 1))), lengths.append(L)
        files.append(fi), offsets.append(max(0, N - 77)), lengths.append(-1)
    return files, offsets, lengths


def span(idx, files, offsets, lengths, R=None):
    """T that every valid request fits exactly."""
    Ns = lengths_at(idx, R)
    return sum(r4(Ns[f] - o if ln == -1 else min(ln, Ns[f] - o)) for f, o, ln in zip(files, offsets, lengths)) or 1


# --------------------------------------------------------------------------- 1. against the float64 reference

@gpu
def test_plain_packed_every_path(ctx):
    """A single-rate corpus of 1, 2 and 4 channels (C = 4), every decode path, power and log."""
    import torch
    idx = cb.index(single_rate_files())
    corpus = cb.Corpus(idx, ctx)
    rng = np.random.default_rng(5)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(150, 9000)), rng)
    T = span(idx, files, offsets, lengths)
    pk = corpus.packed(len(files), T, dtype=torch.float32)
    for log_floor in (None, 1e-10):
        mb = corpus.mel_packed(len(files), T, n_fft=400, hop_length=160, n_mels=80, log_floor=log_floor)
        assert mb.channels == 4 and mb.stride == corpus.mel_packed_frames_bound(len(files), T, hop_length=160)
        check_call(mb, pk, files, offsets, lengths)


@gpu
def test_bit_for_bit_against_mel_crops(ctx):
    """An excerpt inside its file (offset + L <= N) has the frames of the mel crop of (file, offset) of length L."""
    import torch
    idx = cb.index(single_rate_files())
    corpus = cb.Corpus(idx, ctx)
    rng = np.random.default_rng(8)
    Ns = lengths_at(idx)
    for L, kw in ((4000, dict(n_fft=400, hop_length=160, n_mels=80, log_floor=1e-10)),
                  (1003, dict(n_fft=320, win_length=300, hop_length=100, center=False, n_mels=40))):
        files = [int(f) for f in rng.integers(0, len(idx), 12)]
        offsets = [int(rng.integers(0, Ns[f] - L + 1)) for f in files]
        mc = corpus.mel_crops(len(files), L, **kw)
        mb = corpus.mel_packed(len(files), len(files) * r4(L), **kw)
        want, _ = mc(files, offsets)
        feats, starts, frames, _ = mb(files, offsets, [L] * len(files))
        F = mc.n_frames
        assert frames.tolist() == [F] * len(files)
        for b, st in enumerate(starts.tolist()):
            assert torch.equal(feats[:, :, st:st + F].view(torch.int32), want[b].view(torch.int32)), b


@gpu
@pytest.mark.parametrize("g", range(len(GRID)))
def test_resampled_packed_grid(rctx, g):
    """The mixed-rate corpus at 16 kHz over the mel crop grid: n_fft 8 to 4096, short windows, hops below, at and
    above n_fft, both center modes; whole files and random excerpts around the grid's length."""
    *args, L = GRID[g]
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    rng = np.random.default_rng(g)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(1, 3 * L)), rng, R)
    T = span(idx, files, offsets, lengths, R)
    pk = corpus.packed(len(files), T, sample_rate=R)
    for log_floor in (None, 1e-6):
        mb = corpus.mel_packed(len(files), T, R, **mel_args(*args, log_floor=log_floor))
        check_call(mb, pk, files, offsets, lengths)
    del pk
    gc.collect()
    assert WORST[0] <= 1.0
    print(f"worst error / bound so far: {WORST[0]:.3g}")


# --------------------------------------------------------------------------- 2. lengths, tiles, calls

@gpu
@pytest.mark.parametrize("center", [True, False])
def test_length_edges(rctx, center):
    """n_b in {1, n_fft / 2, n_fft / 2 + 1, n_fft - 1, n_fft}, the empty excerpt at offset N, invalid and non-fitting
    excerpts, and a mono file in a 4-channel corpus: 0 frames exactly where the rule says, and rows the file does not
    have exactly 0 or ln(log_floor)."""
    import torch
    idx = cb.index(single_rate_files())
    corpus = cb.Corpus(idx, rctx)
    Ns = lengths_at(idx)
    n_fft, hop = 400, 160
    files, offsets, lengths = [], [], []
    for fi in (2, 0, 1):  # the mono file first
        for n in (1, n_fft // 2, n_fft // 2 + 1, n_fft - 1, n_fft, 1234):
            files.append(fi), offsets.append(7), lengths.append(n)
        files.append(fi), offsets.append(Ns[fi]), lengths.append(-1)  # empty
    bad = [(len(idx), 0, 5), (0, -1, 5), (0, 0, 0), (1, Ns[1] + 1, -1)]
    for f, o, ln in bad:
        files.append(f), offsets.append(o), lengths.append(ln)
    T = span(idx, files[:len(files) - len(bad)], offsets, lengths)
    files.append(0), offsets.append(0), lengths.append(5000)  # does not fit
    pk = corpus.packed(len(files), T, dtype=torch.float32)
    for log_floor in (None, 1e-10, 3.5):
        mb = corpus.mel_packed(len(files), T, n_fft=n_fft, hop_length=hop, center=center, n_mels=64,
                               log_floor=log_floor)
        dev, starts, frames = check_call(mb, pk, files, offsets, lengths)
        m = n_fft // 2 + 1 if center else n_fft
        for b in range(7):  # the mono file: rows 1 .. 3 are constant
            if frames[b]:
                rows = dev[1:, :, starts[b]:starts[b] + frames[b]]
                assert (rows == np.float32(0.0 if log_floor is None else np.log(log_floor))).all()
        got = frames.tolist()
        expect = [n_frames(n, n_fft, hop, center) for n in pk._lengths[:len(files)].tolist()]
        assert got == expect and got[-5:] == [0] * 5 and mb.status.tolist()[-5:] == [90] * 5
        assert [g > 0 for g in got[:5]] == [n >= m for n in (1, 200, 201, 399, 400)]
        with pytest.raises(ValueError, match=f"excerpt {len(files) - 5}: file index"):
            mb(files, offsets, lengths)
    k = len(files) - 5
    with pytest.raises(ValueError, match=f"excerpt {k}: needs columns \\[{T}, {T + 5000}\\), past max_samples {T}"):
        mb(files[:-5] + files[-1:], offsets[:-5] + offsets[-1:], lengths[:-5] + lengths[-1:])


@gpu
def test_many_excerpts_in_one_tile(rctx):
    """Dozens of excerpts of 1 to 3 frames, so that each tile spans several excerpts and alignment gaps, next to a
    long one; then fewer excerpts, then the same call twice: zeros past the new end, bit-identical calls."""
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    rng = np.random.default_rng(11)
    Ns = lengths_at(idx, R)
    files = [int(f) for f in rng.integers(0, len(idx), 90)] + [0]
    lengths = [int(v) for v in rng.integers(1, 700, 90)] + [-1]
    offsets = [int(rng.integers(0, Ns[f] + 1)) for f in files[:-1]] + [0]
    T = span(idx, files, offsets, lengths, R)
    pk = corpus.packed(len(files), T, sample_rate=R)
    mb = corpus.mel_packed(len(files), T, R, n_fft=512, hop_length=256, n_mels=40, log_floor=1e-8)
    full, _, frames = check_call(mb, pk, files, offsets, lengths)
    assert (frames[:-1] > 0).sum() > 40
    short = (files[5:12], offsets[5:12], lengths[5:12])
    a, _, _ = check_call(mb, pk, *short)
    b, _, _ = check_call(mb, pk, *short)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    fresh = corpus.mel_packed(len(files), T, R, n_fft=512, hop_length=256, n_mels=40, log_floor=1e-8)
    c, _, _ = check_call(fresh, pk, *short)
    assert np.array_equal(a.view(np.int32), c.view(np.int32))
    mb([], check=False)  # count 0
    assert not mb.out.view(torch.int32).any()


# --------------------------------------------------------------------------- 3. corpora, requests on the device

@gpu
def test_host_and_attached_corpora(rctx):
    import torch
    idx = cb.index(mixed_files())
    R = 16000
    rng = np.random.default_rng(2)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(100, 6000)), rng, R)
    T = span(idx, files, offsets, lengths, R)
    dev = cb.Corpus(idx, rctx).mel_packed(len(files), T, R, log_floor=1e-10)
    want = dev(files, offsets, lengths)[0].clone()
    with image_path() as path:
        shared = cb.Corpus.share(idx, path, rctx)
        attached = cb.Corpus.attach(path, rctx)
    for c in (cb.Corpus(idx, rctx, memory="host"), shared, attached):
        mb = c.mel_packed(len(files), T, R, log_floor=1e-10)
        got = mb(files, offsets, lengths)[0]
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), c.memory
        del mb, got
    gc.collect()
    attached.close()
    shared.close()


@gpu
def test_device_drawn_requests_without_sync(rctx):
    """Requests drawn on the GPU, check=False under sync debug mode "error", then checked against the packed batch."""
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R, B, T = 16000, 20, 200000
    nt = torch.tensor(lengths_at(idx, R), device="cuda")
    mb = corpus.mel_packed(B, T, R, log_floor=1e-10)
    gen = torch.Generator(device="cuda").manual_seed(7)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            fi = torch.randint(0, len(idx), (B,), device="cuda", generator=gen)
            off = torch.minimum((torch.rand(B, device="cuda", generator=gen) * (nt[fi] + 1)).long(), nt[fi])
            ln = torch.randint(1, 20000, (B,), device="cuda", generator=gen)
            mb(fi, off, ln, check=False)
            draws.append((fi, off, ln, mb.out.clone()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    pk = corpus.packed(B, T, sample_rate=R)
    for fi, off, ln, feats in draws:
        check_call(mb, pk, fi, off, ln)
        assert torch.equal(mb.out.view(torch.int32), feats.view(torch.int32))


@gpu
def test_launch_counts(rctx):
    """A call launches what its packed batch launches, plus the planner and mel_packed_kernel."""
    import torch
    mixed, one = cb.index(mixed_files()), cb.index(single_rate_files())

    def per_call(batch, *args):
        batch(*args, check=False)
        n0 = rctx.launch_count
        batch(*args, check=False)
        return rctx.launch_count - n0

    B, T = 7, 50000
    for c in (cb.Corpus(mixed, rctx), cb.Corpus(mixed, rctx, memory="host")):
        req = (list(range(B)), [0] * B, [5000] * B)
        assert per_call(c.mel_packed(B, T, 16000), *req) == per_call(c.packed(B, T, sample_rate=16000), *req) + 2
    for c in (cb.Corpus(one, rctx), cb.Corpus(one, rctx, memory="host")):
        req = ([0, 1, 2] * 2, [0] * 6, [5000] * 6)
        assert per_call(c.mel_packed(6, T), *req) == per_call(c.packed(6, T, dtype=torch.float32), *req) + 2


# --------------------------------------------------------------------------- 4. refusals, torchaudio

PARAM_REFUSALS = (dict(n_fft=402), dict(n_fft=401), dict(n_fft=6, win_length=6), dict(n_fft=4100, win_length=400),
                  dict(n_fft=8192, win_length=400), dict(n_fft=14 * 2, win_length=20), dict(win_length=0),
                  dict(win_length=401), dict(hop_length=0), dict(n_mels=0), dict(n_mels=513), dict(flags=4),
                  dict(flags=3, log_floor=0.0), dict(flags=3, log_floor=-1.0), dict(flags=3, log_floor=float("inf")),
                  dict(flags=3, log_floor=float("nan")), dict(log_floor=1e-10), dict(params=False),
                  dict(window=None), dict(fbank=None), dict(window="nan"), dict(fbank="nan"), dict(n=0),
                  dict(n=1 << 30), dict(L=0), dict(R=655351), dict(rates_=None), dict(n_files=2))


@gpu
def test_refusals(rctx):
    """clx_batch_create_mel_packed refuses the parameters clx_batch_create_mel_crops refuses, but no length; the
    mel crop refusals are unchanged."""
    Lb = rctx._L
    idx = cb.index(mixed_files()[:3])
    corpus = cb.Corpus(idx, rctx)
    rates = np.array([f.info.sample_rate for f in idx.files], np.uint32)
    good = dict(n_fft=400, win_length=400, hop_length=160, n_mels=80, flags=cb.MEL_CENTER, log_floor=0.0)
    b = C.c_void_p()

    def create(fn, n=4, L=1000, R=16000, window=True, fbank=True, params=True, rates_=rates, n_files=3, **kw):
        p = {**good, **kw}
        mp = cb._lib.MelParams(p["n_fft"], p["win_length"], p["hop_length"], p["n_mels"], p["flags"], p["log_floor"])
        w = np.ones(max(1, p["win_length"]), np.float32)
        fb = np.ones((p["n_fft"] // 2 + 1, max(1, p["n_mels"])), np.float32)
        if window == "nan":
            w[min(7, w.size - 1)] = np.nan
        if fbank == "nan":
            fb[3, min(5, fb.shape[1] - 1)] = np.inf
        return fn(rctx._h, corpus._h, None if rates_ is None else rates_.ctypes.data, n_files, n, L, R,
                  C.byref(mp) if params else None, w.ctypes.data if window is not None else None,
                  fb.ctypes.data if fbank is not None else None, C.byref(b))

    for fn in (Lb.clx_batch_create_mel_packed, Lb.clx_batch_create_mel_crops):
        for kw in PARAM_REFUSALS + (dict(n=1 << 28, L=1 << 62),):
            assert create(fn, **kw) == 90, (fn, kw)
            assert not b.value
    # lengths: refused by the mel crop batch only
    for kw in (dict(L=200), dict(L=399, flags=0), dict(L=1)):
        assert create(Lb.clx_batch_create_mel_crops, **kw) == 90, kw
        assert create(Lb.clx_batch_create_mel_packed, **kw) == 0, kw
        assert Lb.clx_batch_packed_stride(b) == 0 and Lb.clx_batch_mel_frames(b)
        Lb.clx_batch_destroy(rctx._h, b)
    for kw in (dict(L=201), dict(L=400, flags=0)):
        for fn in (Lb.clx_batch_create_mel_crops, Lb.clx_batch_create_mel_packed):
            assert create(fn, **kw) == 0, kw
            Lb.clx_batch_destroy(rctx._h, b)
    assert create(Lb.clx_batch_create_mel_packed, n_fft=8, win_length=8, n_mels=1, L=8, flags=0, R=0, rates_=None) == 0
    assert Lb.clx_batch_packed_requests(b) and Lb.clx_batch_crop_status(b) and Lb.clx_batch_packed_stride(b) == 4
    Lb.clx_batch_destroy(rctx._h, b)
    assert create(Lb.clx_batch_create_mel_crops) == 0
    assert Lb.clx_batch_mel_frames(b) is None
    Lb.clx_batch_destroy(rctx._h, b)
    mixed = cb.Corpus(cb.index(mixed_files()), rctx)
    with pytest.raises(ValueError, match="sample rates"):
        mixed.mel_packed(4, 1000)
    with pytest.raises(ValueError):
        mixed.mel_packed(4, 1000, 16000, mel_scale="kaldi")
    batch = mixed.mel_packed(2, 100, 16000)  # no excerpt can have a frame
    assert batch.out.shape == (4, 128, 0)
    feats, starts, frames, lengths = batch([0, 1], None, [100, 100], check=False)
    assert frames.tolist() == [0, 0] and starts.tolist() == [0, 0] and lengths.tolist() == [100, 0]
    assert batch.status.tolist() == [0, 90]
    del batch, feats, starts, frames, lengths
    gc.collect()
    mixed.close()


@gpu
def test_against_torchaudio(rctx):
    """torchaudio.transforms.MelSpectrogram on the GPU, applied to each excerpt's slice of the packed output, within
    the mel crop tests' bound (with torchaudio's own float32 filterbank)."""
    torch = pytest.importorskip("torch")
    T_ = pytest.importorskip("torchaudio")
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    rng = np.random.default_rng(4)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(300, 20000)), rng, R, n=2)
    T = span(idx, files, offsets, lengths, R)
    pk = corpus.packed(len(files), T, sample_rate=R)
    mb = corpus.mel_packed(len(files), T, R)
    x, s, n = pk(files, offsets, lengths, check=False)
    feats, starts, frames, _ = mb(files, offsets, lengths, check=False)
    ms = T_.transforms.MelSpectrogram(R).cuda()
    fb_ta = T_.functional.melscale_fbanks(201, 0.0, 8000.0, 128, R, None, "htk")
    fb_diff = np.abs(fb_ta.double().numpy() - mb.fbank.astype(np.float64))
    p, checked = mb.params, 0
    for b in range(len(files)):
        F = int(frames[b])
        if not F:
            continue
        seg = x[:, int(s[b]):int(s[b]) + int(n[b])]
        ref = ms(seg).cpu().double().numpy()
        seg = seg.cpu().numpy()
        pw = S.power(seg, p.n_fft, p.hop_length, mb.window, True)
        tol = 2 * S.bound(seg, p.n_fft, p.hop_length, mb.window, mb.fbank, True) + np.swapaxes(pw @ fb_diff, -1, -2)
        got = feats[:, :, int(starts[b]):int(starts[b]) + F].cpu().double().numpy()
        assert got.shape == ref.shape
        err = np.abs(got - ref)
        assert (err <= tol).all(), (b, (err / np.maximum(tol, 1e-30)).max())
        checked += 1
    assert checked > len(idx)
