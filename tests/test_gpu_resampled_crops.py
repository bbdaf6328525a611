"""Resampled crop batches: Corpus.crops(..., sample_rate=R) and clx_batch_create_resampled_crops (-m gpu).

Every crop is compared with tests/spec_resample.py (float64) applied to load() of its whole file: at most 1e-5 apart,
lengths exact, and the columns past a crop's length and the rows its file does not have exactly 0.  A file already at R
must give what a plain CropBatch gives, bit for bit; host corpora and attached images what a device corpus gives.
Statuses are compared with load_crops() of each crop's source span alone.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from tests import spec_resample as S
from tests.test_gpu_corpus import bits, c4ch_config, damaged_index, flac_of
from tests.test_gpu_shared_corpus import image_path

gpu = pytest.mark.gpu
RATE_CODES = {8000: 4, 16000: 5, 22050: 6, 24000: 7, 44100: 9, 48000: 10, 96000: 11}


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


def cfg_at(cfg, rate):
    cfg.sample_rate_code = RATE_CODES[rate]
    return cfg


def variable():  # variable blocking: 1152-sample blocks, every third one 576
    return synth.SynthConfig(seed=78, n_frames=14, block_size=1152, tail_block_size=576, frames_per_file=3,
                             n_channels=1, bps=16, variable_blocking=1, type_mask=synth.TYPE_FIXED | synth.TYPE_LPC,
                             lpc_min_order=1, lpc_max_order=8, rice_mode=-1)


def mono(n_frames, block, seed):
    cfg = synth.workload_config("c2", n_frames, seed)
    cfg.n_channels, cfg.block_size, cfg.stereo_mode = 1, block, synth.INDEPENDENT
    return cfg


_files = {}


def mixed_files():
    """Files at 8 to 96 kHz, of 1, 2 and 4 channels, fixed and variable block sizes (C = 4)."""
    if "mixed" not in _files:
        _files["mixed"] = [
            flac_of(cfg_at(synth.workload_config("c2", 9), 44100)),
            flac_of(cfg_at(synth.workload_config("c2", 7, seed=21), 48000)),
            flac_of(cfg_at(variable(), 8000)),
            flac_of(cfg_at(c4ch_config(), 96000)),
            flac_of(cfg_at(mono(5, 4096, 31), 16000)),
            flac_of(cfg_at(synth.workload_config("c4", 7), 22050)),
            flac_of(cfg_at(mono(6, 1152, 41), 24000)),
        ]
    return _files["mixed"]


class Reference:
    """spec_resample of load() of each file, at each target rate, computed once."""

    def __init__(self, srcs, idx, ctx):
        self.x = [cb.load(s, ctx=ctx)[0].double().cpu().numpy() for s in srcs]
        self.rates = [f.info.sample_rate for f in idx.files]
        self.y = {}

    def full(self, fi, R):
        if (fi, R) not in self.y:
            self.y[fi, R] = S.resample(self.x[fi], self.rates[fi], R)
        return self.y[fi, R]

    def n_t(self, fi, R):
        return S.out_len(self.x[fi].shape[1], self.rates[fi], R)


def check_crops(batch, ref, files, offsets, R, invalid=()):
    """One call of `batch` against the reference; returns (out, lengths, status) on the host."""
    out, lengths = batch(files, offsets, check=False)
    out, lengths, status = out.cpu().numpy(), lengths.cpu().numpy(), batch.status.cpu().numpy()
    L = batch.num_frames
    for b, (fi, o) in enumerate(zip(files, offsets)):
        if b in invalid:
            assert status[b] == 90 and lengths[b] == 0 and not out[b].view(np.int32).any(), b
            continue
        y = ref.full(fi, R)
        m = max(0, min(L, y.shape[1] - o))
        assert lengths[b] == m and status[b] == 0, (b, fi, o, lengths[b], m)
        ch = y.shape[0]
        err = np.abs(out[b, :ch, :m] - y[:, o:o + m]).max(initial=0.0)
        assert err <= 1e-5, (b, fi, o, L, R, err)
        assert not out[b, :ch, m:].view(np.int32).any(), (b, "columns past the length")
        assert not out[b, ch:].view(np.int32).any(), (b, "rows the file lacks")
    return out, lengths, status


def edge_requests(ref, R, n_files, L):
    """Per file: offsets 0, n - 1, n, N_t - 1, N_t, three random ones and one whose crop ends at N_t."""
    rng = np.random.default_rng(R + L)
    files, offsets = [], []
    for fi in range(n_files):
        o_, n, _, _ = S.params(ref.rates[fi], R)
        Nt = ref.n_t(fi, R)
        cand = {0, n - 1, n, max(0, Nt - 1), Nt, max(0, Nt - L)} | set(int(v) for v in rng.integers(0, Nt + 1, 3))
        for o in sorted(c for c in cand if 0 <= c <= Nt):
            files.append(fi)
            offsets.append(o)
    perm = rng.permutation(len(files))
    return [files[p] for p in perm], [offsets[p] for p in perm]


# --------------------------------------------------------------------------- 1. against the float64 reference

@gpu
@pytest.mark.parametrize("R", [16000, 44100, 48000])
def test_mixed_rates_match_reference(rctx, R):
    """One corpus of seven rates in one batch, L from 1 to longer than the shortest file; host corpora and
    attached images give the device corpus's results bit for bit."""
    import torch
    srcs = mixed_files()
    idx = cb.index(srcs)
    ref = Reference(srcs, idx, rctx)
    corpus, host = cb.Corpus(idx, rctx), cb.Corpus(idx, rctx, memory="host")
    shortest = min(ref.n_t(fi, R) for fi in range(len(idx)))
    for L in (1, 3, 37, 1000, 4099, shortest + 5):
        files, offsets = edge_requests(ref, R, len(idx), L)
        batch = corpus.crops(len(files), L, sample_rate=R)
        assert batch.out.shape == (len(files), 4, L) and batch.out.dtype == torch.float32
        out, lengths, status = check_crops(batch, ref, files, offsets, R)
        hbatch = host.crops(len(files), L, sample_rate=R)
        ho, hl = hbatch(files, offsets, check=False)
        assert np.array_equal(ho.cpu().numpy().view(np.int32), out.view(np.int32)) and np.array_equal(hl.cpu(), lengths)
        assert torch.equal(hbatch.status, batch.status) and torch.equal(hbatch._error, batch._error)
    del batch, hbatch
    gc.collect()


@gpu
def test_attached_image_matches_device_corpus(rctx):
    srcs = mixed_files()
    idx = cb.index(srcs)
    ref = Reference(srcs, idx, rctx)
    with image_path() as path:
        shared = cb.Corpus.share(idx, path, rctx)
        attached = cb.Corpus.attach(path, rctx)
    corpus = cb.Corpus(idx, rctx)
    files, offsets = edge_requests(ref, 16000, len(idx), 777)
    out, lengths, _ = check_crops(corpus.crops(len(files), 777, sample_rate=16000), ref, files, offsets, 16000)
    for c in (shared, attached):
        batch = c.crops(len(files), 777, sample_rate=16000)
        o2, l2 = batch(files, offsets)
        assert np.array_equal(o2.cpu().numpy().view(np.int32), out.view(np.int32)) and np.array_equal(l2.cpu(), lengths)
        del batch, o2, l2
    gc.collect()
    attached.close()
    shared.close()


@gpu
@pytest.mark.parametrize("R", [1000, 50])
def test_large_ratios(rctx, R):
    """96 kHz to R: at 1000 Hz the tile shrinks until its source samples fit in shared memory, at 50 Hz one output's
    taps do not fit and the kernel reads the packed output directly."""
    srcs = [flac_of(cfg_at(c4ch_config(), 96000)), flac_of(cfg_at(synth.workload_config("c2", 9), 44100))]
    idx = cb.index(srcs)
    ref = Reference(srcs, idx, rctx)
    corpus = cb.Corpus(idx, rctx)
    for L in (1, 5, 300):
        files, offsets = edge_requests(ref, R, len(idx), L)
        check_crops(corpus.crops(len(files), L, sample_rate=R), ref, files, offsets, R)


# --------------------------------------------------------------------------- 2. files at the target rate

@gpu
def test_same_rate_is_a_crop_batch(ctx, golden):
    """At R equal to a file's rate the crop is copied: out, lengths, status and the error word are a CropBatch's, bit
    for bit, on every decode path, invalid requests included."""
    import torch
    srcs = mixed_files()
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    for R, fi in ((44100, 0), (48000, 1), (8000, 2)):
        N = idx[fi].length
        offsets = [0, 1, 5, N // 3, N - 4097, N - 1, N, N + 1, -1, 0, 17]
        files = [fi] * 9 + [len(idx), (1 << 32) + fi]
        for L in (1, 4096, N + 3):
            a, b = corpus.crops(len(files), L, dtype=torch.float32), corpus.crops(len(files), L, sample_rate=R)
            oa, la = a(files, offsets, check=False)
            ob, lb = b(files, offsets, check=False)
            assert torch.equal(bits(oa), bits(ob)) and torch.equal(la, lb), (R, L)
            assert torch.equal(a.status, b.status) and torch.equal(a._error, b._error), (R, L)
            assert b.status.cpu().tolist()[7:] == [90] * 4
            with pytest.raises(ValueError) as ea:
                a(files, offsets)
            with pytest.raises(ValueError) as eb:
                b(files, offsets)
            assert str(ea.value) == str(eb.value)


# --------------------------------------------------------------------------- 3. edges and invalid requests

@gpu
def test_invalid_requests(rctx):
    import torch
    srcs = mixed_files()
    idx = cb.index(srcs)
    ref = Reference(srcs, idx, rctx)
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    files, offsets = edge_requests(ref, R, len(idx), 300)
    bad = {2: (len(idx), 0), 5: (-1, 0), 9: (0, -1), 12: (1, ref.n_t(1, R) + 1), 14: (3, -(1 << 40)),
           17: ((1 << 32) + 2, 0), 19: (5, ref.n_t(5, R) + 1)}
    for b, (f, o) in bad.items():
        files[b], offsets[b] = f, o
    batch = corpus.crops(len(files), 300, sample_rate=R)
    batch([0] * len(files), [0] * len(files))  # a full crop first: the invalid crops' rows must then be zeroed
    check_crops(batch, ref, files, offsets, R, invalid=set(bad))
    err = int(batch._error.item()) & ((1 << 64) - 1)
    assert err >> 62 == 0 and (err >> 32) & ((1 << 30) - 1) == 2 and err & 0xffffffff == 90
    with pytest.raises(ValueError, match=f"crop 2: file index {len(idx)} out of range"):
        batch(files, offsets)
    one = corpus.crops(1, 300, sample_rate=R)
    with pytest.raises(ValueError, match=f"crop 0: offset {ref.n_t(1, R) + 1} outside file 1 "
                                         f"\\({ref.n_t(1, R)} samples at 16000 Hz\\)"):
        one([1], [ref.n_t(1, R) + 1])
    with pytest.raises(TypeError):
        batch(torch.zeros(len(files)), offsets)


# --------------------------------------------------------------------------- 4. damaged files

@gpu
def test_damaged_files(rctx, golden):
    """Each crop's status is load_crops()'s of its source span alone; check=True raises what the error word names."""
    import torch
    idx = damaged_index(golden)
    corpus = cb.Corpus(idx, rctx)
    R, L = 16000, 3000
    files, offsets = [], []
    for fi, f in enumerate(idx.files):
        r = f.info.sample_rate
        Nt = S.out_len(f.length, r, R)
        for o in sorted({0, Nt // 4, Nt // 2, max(0, Nt - L), max(0, Nt - 10), Nt}):
            files.append(fi)
            offsets.append(o)
    batch = corpus.crops(len(files), L, sample_rate=R)
    batch(files, offsets, check=False)
    st = batch.status.cpu().tolist()
    for b, (fi, o) in enumerate(zip(files, offsets)):
        lo, hi = S.source_span(idx[fi].length, idx[fi].info.sample_rate, R, o, L)
        try:
            cb.load_crops(idx, [fi], [lo], max(1, hi - lo), dtype=torch.float32, ctx=rctx)
            want = 0
        except cb.Error as e:
            want = e.status
        assert st[b] == want, (b, fi, o, lo, hi)
    assert any(st)
    err = int(batch._error.item()) & ((1 << 64) - 1)
    b = (err >> 32) & ((1 << 30) - 1)
    with pytest.raises(cb.Error) as e:
        batch(files, offsets)
    assert e.value.status == st[b] != 0 and f"(file {files[b]}, crop {b})" in str(e.value)


# --------------------------------------------------------------------------- 5. device-drawn requests, launches

@gpu
def test_device_drawn_requests_without_sync(rctx):
    """Requests drawn on the GPU, check=False under sync debug mode "error"; two batches of one corpus interleaved, a
    long crop batch before a short one."""
    import torch
    srcs = mixed_files()
    idx = cb.index(srcs)
    ref = Reference(srcs, idx, rctx)
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    nt = torch.tensor([ref.n_t(fi, R) for fi in range(len(idx))], device="cuda")
    a, b = corpus.crops(24, 20000, sample_rate=R), corpus.crops(16, 77, sample_rate=R)
    gen = torch.Generator(device="cuda").manual_seed(5)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(3):
            for batch in (a, b):
                fi = torch.randint(0, len(idx), (batch.batch,), device="cuda", generator=gen)
                off = (torch.rand(batch.batch, device="cuda", generator=gen) * (nt[fi] + 1)).long()
                off = torch.minimum(off, nt[fi])
                batch(fi, off, check=False)
                draws.append((batch, fi, off, batch.out.clone(), batch.lengths.clone(), batch.status.clone()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for batch, fi, off, out, lengths, status in draws:
        assert not status.any()
        L, out, lengths = batch.num_frames, out.cpu().numpy(), lengths.cpu().numpy()
        for k, (f, o) in enumerate(zip(fi.tolist(), off.tolist())):
            y = ref.full(f, R)
            m = max(0, min(L, y.shape[1] - o))
            assert lengths[k] == m
            assert np.abs(out[k, :y.shape[0], :m] - y[:, o:o + m]).max(initial=0.0) <= 1e-5
            assert not out[k, :y.shape[0], m:].any() and not out[k, y.shape[0]:].any()


@gpu
def test_launch_counts(rctx):
    """A call launches what the packed batch of its source spans launches, plus the map and filter kernels."""
    import torch
    srcs = mixed_files()
    idx = cb.index(srcs)
    dev, host = cb.Corpus(idx, rctx), cb.Corpus(idx, rctx, memory="host")

    def per_call(batch, *args):
        batch(*args, check=False)
        n0 = rctx.launch_count
        batch(*args, check=False)
        return rctx.launch_count - n0

    B, L, R = 7, 5000, 16000
    T = B * ((dev.resample_source_bound(L, R) + 3) & ~3)
    for c in (dev, host):
        packed = per_call(c.packed(B, T, dtype=torch.float32), list(range(B)))
        resampled = per_call(c.crops(B, L, sample_rate=R), list(range(B)), [0] * B)
        assert resampled == packed + 2, (c.memory, packed, resampled)


# --------------------------------------------------------------------------- 6. refusals

@gpu
def test_refusals(rctx):
    import torch
    L = rctx._L
    srcs = mixed_files()[:3]
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, rctx)
    h = corpus._h
    b = C.c_void_p()

    def create(rates, n_crops=4, L_=100, R=16000, n_files=None):
        arr = np.array(rates, dtype=np.uint32)
        return L.clx_batch_create_resampled_crops(rctx._h, h, arr.ctypes.data, len(rates) if n_files is None else n_files,
                                                  n_crops, L_, R, C.byref(b))

    good = [44100, 48000, 8000]
    for args in (([0, 48000, 8000],), ([44100, 655351, 8000],), (good, 4, 100, 0), (good, 4, 100, 655351),
                 (good, 0), (good, 4, 0), (good, 1 << 30), (good, 4, 1 << 62), (good[:2],), (good, 4, 100, 16000, 4),
                 ([655347, 655343, 8000], 4, 100, 655349)):  # 2 x 655349 phases x 13 taps > 2^24 coefficients
        assert create(*args) == 90, args
        assert not b.value
    assert L.clx_batch_create_resampled_crops(rctx._h, h, None, 3, 4, 100, 16000, C.byref(b)) == 90
    assert create([655347, 655349, 655349], 4, 100, 655349) == 0  # one such table fits
    L.clx_batch_destroy(rctx._h, b)
    assert create([655350, 1, 8000], 2, 3, 655350) == 0  # the limits themselves
    assert L.clx_batch_crop_requests(b) and L.clx_batch_packed_requests(b) is None
    assert L.clx_corpus_destroy(rctx._h, h) == 90  # a live batch
    L.clx_batch_destroy(rctx._h, b)
    # frames above 24 bits cannot be float32
    data = flac_of(synth.workload_config("c2", 8))
    wide = cb.index(data)[0].descs.copy()
    wide["bits_per_sample"][5] = 25
    ff = np.array([0, 4, 8], np.uint32)
    hw = C.c_void_p()
    assert L.clx_corpus_create(rctx._h, data.ctypes.data, data.size, wide.ctypes.data, wide.size, ff.ctypes.data, 2,
                               C.byref(hw)) == 0
    rates = np.array([44100, 44100], np.uint32)
    assert L.clx_batch_create_resampled_crops(rctx._h, hw, rates.ctypes.data, 2, 4, 100, 16000, C.byref(b)) == 90
    assert L.clx_corpus_destroy(rctx._h, hw) == 0
    with pytest.raises(ValueError):
        corpus.crops(4, 100, dtype=torch.int32, sample_rate=16000)
    with pytest.raises(cb.Error):
        corpus.crops(4, 100, sample_rate=0)
    batch = corpus.crops(2, 10, sample_rate=16000)
    with pytest.raises(cb.Error):
        corpus.close()
    del batch
    gc.collect()
    corpus.close()
