"""Resampled packed batches: Corpus.packed(..., sample_rate=R) and clx_batch_create_resampled_packed (-m gpu).

Every excerpt is compared with tests/spec_resample.py (float64) applied to load() of its whole file: at most 1e-5 apart,
starts and lengths exact, and every element of the [C, stride] output that no excerpt covers exactly 0 (as int32 bits).
A corpus whose files are all at R must give what a plain float32 PackedBatch gives, bit for bit; host corpora and
attached images what a device corpus gives.  Statuses are compared with load_crops() of each excerpt's source span.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from tests import spec_resample as S
from tests.test_gpu_corpus import bits, c4ch_config, damaged_index, flac_of
from tests.test_gpu_resampled_crops import Reference, cfg_at, mixed_files, variable
from tests.test_gpu_shared_corpus import image_path

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


def r4(n):
    return (n + 3) & ~3


def layout(ref, files, offsets, lengths, T, R):
    """Per request (start, n_b), n_b None for an invalid request or an excerpt that does not fit."""
    out, at = [], 0
    for fi, o, ln in zip(files, offsets, lengths):
        if not 0 <= fi < len(ref.x) or ln == 0 or ln < -1:
            out.append((at, None))
            continue
        Nt = ref.n_t(fi, R)
        if not 0 <= o <= Nt:
            out.append((at, None))
            continue
        n = Nt - o if ln == -1 else min(ln, Nt - o)
        out.append((at, n if at + n <= T else None))
        at += r4(n)
    return out


def full_out(batch):
    """The whole [C, stride] output, [T, stride) included."""
    return batch.out.as_strided((batch.channels, batch.stride), (batch.stride, 1))


def check_call(batch, ref, files, offsets, lengths, R):
    """One call of `batch` (check=False) against the reference; returns (out [C, stride], starts, lengths, status)."""
    out, st, ln = batch(files, offsets, lengths, check=False)
    T = batch.max_samples
    assert out.shape == (batch.channels, T)
    want = layout(ref, files, offsets, lengths, T, R)
    full = full_out(batch).cpu().numpy()
    st, ln, status = st.cpu().numpy(), ln.cpu().numpy(), batch.status.cpu().numpy()
    assert st.tolist() == [s for s, _ in want]
    assert ln.tolist() == [n or 0 for _, n in want]
    assert status.tolist() == [0 if n is not None else 90 for _, n in want]
    covered = np.zeros(full.shape, dtype=bool)
    for b, ((s, n), fi, o) in enumerate(zip(want, files, offsets)):
        if not n:
            continue
        y = ref.full(fi, R)
        ch = y.shape[0]
        err = np.abs(full[:ch, s:s + n] - y[:, o:o + n]).max(initial=0.0)
        assert err <= 1e-5, (b, fi, o, n, R, err)
        covered[:ch, s:s + n] = True
    stray = np.nonzero(full.view(np.int32) * ~covered)
    assert stray[0].size == 0, ("uncovered elements not 0", stray[0][:4], stray[1][:4])
    return full, st, ln, status


def mixed(rctx):
    srcs = mixed_files()
    idx = cb.index(srcs)
    return srcs, idx, Reference(srcs, idx, rctx)


# --------------------------------------------------------------------------- 1. whole files and excerpts

@gpu
@pytest.mark.parametrize("R", [16000, 44100, 48000])
def test_whole_files_match_reference(rctx, R):
    """Every file of a seven-rate corpus whole (length -1): lengths N_t, starts the round_up_4 scan; a host corpus
    gives the device corpus's results bit for bit."""
    import torch
    srcs, idx, ref = mixed(rctx)
    k = len(idx)
    corpus, host = cb.Corpus(idx, rctx), cb.Corpus(idx, rctx, memory="host")
    T = sum(r4(ref.n_t(fi, R)) for fi in range(k)) + 5
    batch, hbatch = corpus.packed(k + 2, T, sample_rate=R), host.packed(k + 2, T, sample_rate=R)
    assert batch.out.dtype == torch.float32 and batch.stride == r4(T)
    files = list(range(k))[::-1]
    full, st, ln, status = check_call(batch, ref, files, [0] * k, [-1] * k, R)
    assert ln.tolist() == [ref.n_t(fi, R) for fi in files]
    ho, hs, hl = hbatch(files, None, None, check=False)
    assert np.array_equal(full_out(hbatch).cpu().numpy().view(np.int32), full.view(np.int32))
    assert np.array_equal(hs.cpu(), st) and np.array_equal(hl.cpu(), ln)
    assert torch.equal(hbatch.status, batch.status) and torch.equal(hbatch._error, batch._error)
    batch(files)  # check=True raises nothing


@gpu
def test_against_torchaudio(rctx):
    """One call against torchaudio.functional.resample itself, on float64 input."""
    import torch
    F = pytest.importorskip("torchaudio.functional")
    srcs, idx, ref = mixed(rctx)
    R, k = 16000, len(idx)
    batch = cb.Corpus(idx, rctx).packed(k, sum(r4(ref.n_t(fi, R)) for fi in range(k)), sample_rate=R)
    out, starts, lengths = batch(list(range(k)))
    for fi in range(k):
        y = F.resample(torch.from_numpy(ref.x[fi]), ref.rates[fi], R).numpy()
        s, n = int(starts[fi]), int(lengths[fi])
        assert n == y.shape[1]
        assert np.abs(out[:y.shape[0], s:s + n].cpu().numpy() - y).max() <= 1e-5, fi


@gpu
def test_random_excerpts(rctx):
    """Offsets 0, n - 1, n, N_t - 1 and N_t; lengths 1, 2, 3, n and several tiles; dozens of 1-7 sample excerpts in one
    tile next to one excerpt longer than many tiles."""
    srcs, idx, ref = mixed(rctx)
    corpus = cb.Corpus(idx, rctx)
    rng = np.random.default_rng(3)
    for R in (16000, 48000):
        files, offsets, lengths = [], [], []
        for fi in range(len(idx)):
            _, n, _, _ = S.params(ref.rates[fi], R)
            Nt = ref.n_t(fi, R)
            for o in sorted({0, n - 1, n, max(0, Nt - 1), Nt, int(rng.integers(0, Nt + 1))}):
                for ln in (1, 2, 3, n, 2500, 5000, -1):
                    if o <= Nt:
                        files.append(fi)
                        offsets.append(o)
                        lengths.append(ln)
        perm = rng.permutation(len(files))
        files, offsets, lengths = ([x[p] for p in perm] for x in (files, offsets, lengths))
        T = sum(r4(n or 0) for _, n in layout(ref, files, offsets, lengths, 1 << 40, R))
        check_call(corpus.packed(len(files), T, sample_rate=R), ref, files, offsets, lengths, R)
        # short excerpts crowding tiles, then one long one
        files = [int(f) for f in rng.integers(0, len(idx), 120)] + [1]
        offsets = [int(rng.integers(0, ref.n_t(f, R))) for f in files[:-1]] + [0]
        lengths = [int(v) for v in rng.integers(1, 8, 120)] + [-1]
        T = sum(r4(n) for _, n in layout(ref, files, offsets, lengths, 1 << 40, R))
        check_call(corpus.packed(len(files), T, sample_rate=R), ref, files, offsets, lengths, R)


# --------------------------------------------------------------------------- 2. capacity

@gpu
def test_capacity(rctx):
    """An exact fit at T, one sample over, the refused suffix, count 0, count = max_excerpts, and a long call then a
    short one against a fresh batch."""
    import torch
    srcs, idx, ref = mixed(rctx)
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    files, lengths = [0, 2, 3, 1, 5], [1000, 777, -1, 5, 3001]
    offsets = [10, 0, 0, 3, 100]
    need = layout(ref, files, offsets, lengths, 1 << 40, R)
    exact = need[-1][0] + need[-1][1]
    for T in (exact, exact - 1, exact + 1, need[2][0] + 3):
        batch = corpus.packed(len(files), T, sample_rate=R)
        _, _, ln, status = check_call(batch, ref, files, offsets, lengths, R)
        if T == exact - 1:
            assert status.tolist()[-1] == 90
            with pytest.raises(ValueError, match=f"excerpt 4: needs columns \\[{need[4][0]}, {exact}\\) at 16000 Hz, "
                                                 f"past max_samples {T}"):
                batch(files, offsets, lengths)
        if T == need[2][0] + 3:  # the refused suffix
            assert status.tolist() == [0, 0, 90, 90, 90]
    batch = corpus.packed(len(files), exact, sample_rate=R)
    check_call(batch, ref, files, offsets, lengths, R)  # count = max_excerpts
    out, st, ln = batch([], check=False)  # count 0
    assert st.numel() == 0 and not bits(full_out(batch)).any()
    # a long call, then a short one: the same as a fresh batch's short call
    check_call(batch, ref, files, offsets, lengths, R)
    short = ([4, 6], [7, 0], [50, 9])
    a, _, _, _ = check_call(batch, ref, *short, R)
    fresh = corpus.packed(len(files), exact, sample_rate=R)
    b, _, _, _ = check_call(fresh, ref, *short, R)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    assert torch.equal(batch._error, fresh._error)


# --------------------------------------------------------------------------- 3. files at the target rate

def at_r_files(rate):
    return [flac_of(cfg_at(synth.workload_config("c2", 9), rate)), flac_of(cfg_at(c4ch_config(), rate)),
            flac_of(cfg_at(variable(), rate))]


@gpu
def test_same_rate_is_a_packed_batch(ctx):
    """A corpus whose files are all at R: out, starts, lengths, status and the error word are a float32 PackedBatch's,
    bit for bit, on every decode path, invalid and non-fitting requests included; so are the raises."""
    import torch
    srcs = at_r_files(44100)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    N = [f.length for f in idx.files]
    files = [0, 1, 2, 0, 1, 3, 2, 0, -1, 1, (1 << 32) + 1, 2]
    offsets = [0, 5, N[2] - 1, N[0], N[1] + 1, 0, 17, 3, 0, 0, 0, -2]
    lengths = [-1, 4097, 3, 8, -1, 1, 0, -2, 5, 1000, 5, 4]
    for T in (1, 4099, sum(r4(n) for n in N) + 7, 2 * sum(N)):
        a = corpus.packed(len(files), T, dtype=torch.float32)
        b = corpus.packed(len(files), T, sample_rate=44100)
        assert a.stride >= b.stride == r4(T)
        for args in ((files, offsets, lengths), (files[:3], None, None), ([2, 0], [N[2] - 2, 1], [9, 9])):
            oa, sa, la = a(*args, check=False)
            ob, sb, lb = b(*args, check=False)
            assert torch.equal(bits(oa), bits(ob)) and torch.equal(sa, sb) and torch.equal(la, lb), (T, args)
            assert torch.equal(a.status, b.status) and torch.equal(a._error, b._error), (T, args)
            assert not bits(full_out(b)[:, T:]).any()
        with pytest.raises(ValueError) as ea:
            a(files, offsets, lengths)
        with pytest.raises(ValueError) as eb:
            b(files, offsets, lengths)
        assert str(ea.value) == str(eb.value)


@gpu
def test_files_at_r_in_a_mixed_corpus(rctx):
    """In the seven-rate corpus, the excerpts of the files at R are the plain batch's columns, bit for bit."""
    import torch
    srcs, idx, ref = mixed(rctx)
    corpus = cb.Corpus(idx, rctx)
    for R, fi in ((44100, 0), (48000, 1), (16000, 4)):
        N = idx[fi].length
        offsets, lengths = [0, 1, N // 3, N - 5, N], [-1, 4096, 3, 9, 4]
        files = [fi] * len(offsets)
        T = 2 * N + 64
        a = corpus.packed(len(files), T, dtype=torch.float32)
        b = corpus.packed(len(files), T, sample_rate=R)
        oa, sa, la = a(files, offsets, lengths)
        ob, sb, lb = b(files, offsets, lengths)
        assert torch.equal(sa, sb) and torch.equal(la, lb) and torch.equal(a.status, b.status)
        assert torch.equal(bits(oa), bits(ob)), R


# --------------------------------------------------------------------------- 4. large ratios, host corpora, images

@gpu
@pytest.mark.parametrize("R", [1000, 50])
def test_large_ratios(rctx, R):
    """96 kHz to R: at 1000 Hz the tile shrinks until its source samples fit in shared memory, at 50 Hz one output's
    taps do not fit and the kernel reads the packed output directly."""
    srcs = [flac_of(cfg_at(c4ch_config(), 96000)), flac_of(cfg_at(synth.workload_config("c2", 9), 44100))]
    idx = cb.index(srcs)
    ref = Reference(srcs, idx, rctx)
    corpus = cb.Corpus(idx, rctx)
    files, offsets, lengths = [0, 1, 0, 1, 0, 1], [0, 0, 1, 2, ref.n_t(0, R) - 1, 3], [-1, -1, 1, 5, -1, 300]
    T = sum(r4(n) for _, n in layout(ref, files, offsets, lengths, 1 << 40, R))
    check_call(corpus.packed(len(files), T, sample_rate=R), ref, files, offsets, lengths, R)


@gpu
def test_host_and_attached_match_device(rctx):
    import torch
    srcs, idx, ref = mixed(rctx)
    R = 16000
    rng = np.random.default_rng(9)
    files = [int(f) for f in rng.integers(0, len(idx), 40)]
    offsets = [int(rng.integers(0, ref.n_t(f, R) + 1)) for f in files]
    lengths = [int(v) for v in rng.choice([-1, 1, 7, 300, 4000], 40)]
    T = 60000
    corpus = cb.Corpus(idx, rctx)
    dev = corpus.packed(len(files), T, sample_rate=R)
    full, st, ln, status = check_call(dev, ref, files, offsets, lengths, R)
    with image_path() as path:
        shared = cb.Corpus.share(idx, path, rctx)
        attached = cb.Corpus.attach(path, rctx)
    host = cb.Corpus(idx, rctx, memory="host")
    for c in (host, shared, attached):
        batch = c.packed(len(files), T, sample_rate=R)
        o2, s2, l2 = batch(files, offsets, lengths, check=False)
        assert np.array_equal(full_out(batch).cpu().numpy().view(np.int32), full.view(np.int32)), c.memory
        assert np.array_equal(s2.cpu(), st) and np.array_equal(l2.cpu(), ln)
        assert torch.equal(batch.status, dev.status) and torch.equal(batch._error, dev._error)
        del batch, o2, s2, l2
    gc.collect()
    attached.close()
    shared.close()


# --------------------------------------------------------------------------- 5. damaged files

@gpu
def test_damaged_files(rctx, golden):
    """Each excerpt's status is load_crops()'s of its source span alone; check=True raises, in excerpt order, ValueError
    for an invalid request before a failed excerpt, else the Error the error word names."""
    import torch
    idx = damaged_index(golden)
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    files, offsets, lengths = [], [], []
    for fi, f in enumerate(idx.files):
        Nt = S.out_len(f.length, f.info.sample_rate, R)
        for o, ln in ((0, -1), (Nt // 4, 3000), (Nt // 2, 5), (max(0, Nt - 3000), -1), (max(0, Nt - 10), 4), (Nt, 2)):
            files.append(fi)
            offsets.append(o)
            lengths.append(ln)
    T = 1 << 22
    batch = corpus.packed(len(files), T, sample_rate=R)
    _, _, ln = batch(files, offsets, lengths, check=False)
    st, ln = batch.status.cpu().tolist(), ln.cpu().tolist()
    for b, (fi, o) in enumerate(zip(files, offsets)):
        f = idx[fi]
        lo, hi = S.source_span(f.length, f.info.sample_rate, R, o, ln[b])
        try:
            cb.load_crops(idx, [fi], [lo], max(1, hi - lo), dtype=torch.float32, ctx=rctx)
            want = 0
        except cb.Error as e:
            want = e.status
        assert st[b] == want, (b, fi, o, lo, hi)
    assert any(st)
    err = int(batch._error.item()) & ((1 << 64) - 1)
    first = (err >> 32) & ((1 << 30) - 1)
    assert first == min(b for b, s in enumerate(st) if s)
    with pytest.raises(cb.Error) as e:
        batch(files, offsets, lengths)
    assert e.value.status == st[first] != 0 and f"(file {files[first]}, excerpt {first})" in str(e.value)
    # an invalid request before the first failed excerpt: ValueError
    bad, r = list(offsets), idx[files[0]].info.sample_rate
    bad[0] = S.out_len(idx[files[0]].length, r, R) + 1
    at = "" if r == R else " at 16000 Hz"
    with pytest.raises(ValueError, match=f"excerpt 0: offset {bad[0]} outside file {files[0]} "
                                         f"\\({bad[0] - 1} samples{at}\\)"):
        batch(files, bad, lengths)


# --------------------------------------------------------------------------- 6. device-drawn requests, launches

@gpu
def test_device_drawn_requests_without_sync(rctx):
    """Requests drawn on the GPU, check=False under sync debug mode "error"; two batches of one corpus interleaved."""
    import torch
    srcs, idx, ref = mixed(rctx)
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    nt = torch.tensor([ref.n_t(fi, R) for fi in range(len(idx))], device="cuda")
    a, b = corpus.packed(24, 200000, sample_rate=R), corpus.packed(16, 3000, sample_rate=R)
    gen = torch.Generator(device="cuda").manual_seed(5)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(3):
            for batch in (a, b):
                n = batch.max_excerpts - it
                fi = torch.randint(0, len(idx), (n,), device="cuda", generator=gen)
                off = torch.minimum((torch.rand(n, device="cuda", generator=gen) * (nt[fi] + 1)).long(), nt[fi])
                ln = torch.randint(-1, 9000, (n,), device="cuda", generator=gen)
                ln = torch.where(ln == 0, torch.ones_like(ln), ln)
                out, st, lens = batch(fi, off, ln, check=False)
                draws.append((batch, fi, off, ln, full_out(batch).clone(), st.clone(), lens.clone(),
                              batch.status.clone()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for batch, fi, off, ln, full, st, lens, status in draws:
        files, offsets, lengths = fi.tolist(), off.tolist(), ln.tolist()
        want = layout(ref, files, offsets, lengths, batch.max_samples, R)
        assert st.tolist() == [s for s, _ in want] and lens.tolist() == [n or 0 for _, n in want]
        assert status.tolist() == [0 if n is not None else 90 for _, n in want]
        full = full.cpu().numpy()
        covered = np.zeros(full.shape, dtype=bool)
        for (s, n), f, o in zip(want, files, offsets):
            if n:
                y = ref.full(f, R)
                assert np.abs(full[:y.shape[0], s:s + n] - y[:, o:o + n]).max() <= 1e-5
                covered[:y.shape[0], s:s + n] = True
        assert not (full.view(np.int32) * ~covered).any()


@gpu
def test_launch_counts(rctx):
    """A call launches what the inner packed batch launches, plus the map and filter kernels."""
    import torch
    srcs, idx, _ = mixed(rctx)
    dev, host = cb.Corpus(idx, rctx), cb.Corpus(idx, rctx, memory="host")

    def per_call(batch, *args):
        batch(*args, check=False)
        n0 = rctx.launch_count
        batch(*args, check=False)
        return rctx.launch_count - n0

    B, T, R = 7, 50000, 16000
    for c in (dev, host):
        T_src = c.resample_packed_source_bound(B, T, R)
        assert T_src >= T * 96000 // R
        packed = per_call(c.packed(B, T_src, dtype=torch.float32), list(range(B)))
        resampled = per_call(c.packed(B, T, sample_rate=R), list(range(B)))
        assert resampled == packed + 2, (c.memory, packed, resampled)


# --------------------------------------------------------------------------- 7. refusals

@gpu
def test_refusals(rctx):
    import torch
    L = rctx._L
    srcs = mixed_files()[:3]
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, rctx)
    h = corpus._h
    b = C.c_void_p()

    def create(rates, B=4, T=100, R=16000, n_files=None):
        arr = np.array(rates, dtype=np.uint32)
        return L.clx_batch_create_resampled_packed(rctx._h, h, arr.ctypes.data, len(rates) if n_files is None else
                                                   n_files, B, T, R, C.byref(b))

    good = [44100, 48000, 8000]
    for args in (([0, 48000, 8000],), ([44100, 655351, 8000],), (good, 4, 100, 0), (good, 4, 100, 655351),
                 (good, 0), (good, 4, 0), (good, 1 << 30), (good, 4, 1 << 62), (good, 4, 1 << 59, 16000),
                 (good[:2],), (good, 4, 100, 16000, 4),
                 ([655347, 655343, 8000], 4, 100, 655349)):  # 2 x 655349 phases x 13 taps > 2^24 coefficients
        assert create(*args) == 90, args
        assert not b.value
    assert L.clx_batch_create_resampled_packed(rctx._h, h, None, 3, 4, 100, 16000, C.byref(b)) == 90
    assert create([655350, 1, 8000], 2, 3, 655350) == 0  # the limits themselves
    assert L.clx_batch_packed_requests(b) and L.clx_batch_packed_starts(b) and L.clx_batch_packed_count(b)
    assert L.clx_batch_packed_stride(b) == 4 and L.clx_batch_crop_requests(b) is None
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
    assert L.clx_batch_create_resampled_packed(rctx._h, hw, rates.ctypes.data, 2, 4, 100, 16000, C.byref(b)) == 90
    assert L.clx_corpus_destroy(rctx._h, hw) == 0
    with pytest.raises(ValueError):
        corpus.packed(4, 100, dtype=torch.int32, sample_rate=16000)
    with pytest.raises(cb.Error):
        corpus.packed(4, 100, sample_rate=0)
    with pytest.raises(ValueError):
        corpus.packed(0, 100, sample_rate=16000)
    batch = corpus.packed(2, 10, sample_rate=16000)
    with pytest.raises(ValueError, match="3 excerpts for a batch of at most 2"):
        batch([0, 1, 2])
    with pytest.raises(TypeError):
        batch(torch.zeros(2))
    with pytest.raises(cb.Error):
        corpus.close()
    del batch
    gc.collect()
    corpus.close()
