"""Packed batches: Corpus.packed / PackedBatch and the C ABI under them (-m gpu).

Every excerpt is compared bit for bit with load() of the same file (frame_offset=, num_frames=), whose views use the
same layout; the columns between excerpts, past the last one and the rows a file does not have must read 0.  Statuses
and raises are compared with load_crops() of each excerpt alone.  Host corpora are compared with device corpora.
"""
import ctypes as C
import gc
import hashlib

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from tests.test_gpu_batch_out import corruption_corpus
from tests.test_gpu_corpus import bits, damaged_index, files_1_2_4, flac_of, raised

gpu = pytest.mark.gpu


def expected(idx, srcs, files, offsets, lengths, T, dtype, ctx):
    """The [C, T] tensor a call must give, its starts and lengths, from load() of each excerpt (None: does not fit)."""
    import torch
    C_ = max(f.info.channels for f in idx.files)
    out = torch.zeros((C_, T), dtype=dtype, device="cuda")
    starts, lens, at = [], [], 0
    for fi, o, ln in zip(files, offsets, lengths):
        N = idx[fi].length
        n = N - o if ln == -1 else min(ln, N - o)
        starts.append(at)
        if at + n > T:
            lens.append(None)
            at += (n + 3) & ~3
            continue
        if n:
            t, _ = cb.load(srcs[fi], dtype=dtype, ctx=ctx, frame_offset=o, num_frames=n)
            out[:t.shape[0], at:at + n] = t
        lens.append(n)
        at += (n + 3) & ~3
    return out, starts, lens


def check_call(batch, idx, srcs, files, offsets, lengths, ctx, host=None):
    import torch
    T = batch.max_samples
    exp, starts, lens = expected(idx, srcs, files, offsets, lengths, T, batch.dtype, ctx)
    out, st, ln = batch(files, offsets, lengths, check=False)
    fits = [x is not None for x in lens]
    assert st.cpu().tolist() == starts
    assert ln.cpu().tolist() == [x if x is not None else 0 for x in lens]
    assert batch.status.cpu().tolist() == [0 if f else 90 for f in fits]
    assert torch.equal(bits(out), bits(exp)), torch.nonzero(bits(out) != bits(exp))[:4].tolist()
    if host is not None:
        ho, hs, hl = host(files, offsets, lengths, check=False)
        assert torch.equal(bits(ho), bits(out)) and torch.equal(hs, st) and torch.equal(hl, ln)
        assert torch.equal(host.status, batch.status) and torch.equal(host._error, batch._error)
    return out


# --------------------------------------------------------------------------- 1. whole files and excerpts against load()

@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_whole_files_match_load(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    srcs = files_1_2_4(golden)
    idx = cb.index(srcs)
    corpus, host = cb.Corpus(idx, ctx), cb.Corpus(idx, ctx, memory="host")
    k = len(srcs)
    views = cb.load(list(srcs), dtype=dtype, ctx=ctx)
    T = sum((f.length + 3) & ~3 for f in idx.files) + 5
    batch, hbatch = corpus.packed(k + 2, T, dtype=dtype), host.packed(k + 2, T, dtype=dtype)
    out = check_call(batch, idx, srcs, list(range(k)), [0] * k, [-1] * k, ctx, host=hbatch)
    out, starts, lengths = batch(torch.arange(k, device="cuda"))
    assert out.shape == (4, T) and out.dtype == dtype
    for i, (v, _) in enumerate(views):
        s, n = int(starts[i]), int(lengths[i])
        assert n == idx[i].length and s % 4 == 0
        assert torch.equal(bits(out[:v.shape[0], s:s + n]), bits(v)), i
    # the STREAMINFO MD5 of the golden fixtures, out of `out`
    for i, name in ((4, "pop"), (5, "short"), (6, "wasted_bits")):
        si, _ = cb.open_stream(golden[f"{name}__bytes"])
        if dtype == torch.int32:
            s, n = int(starts[i]), int(lengths[i])
            pcm = out[:si.channels, s:s + n].cpu().numpy()
            assert hashlib.md5(pcm.T.astype("<i2").tobytes()).digest() == si.md5sum, name


@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_random_excerpts_match_load(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    srcs = files_1_2_4(golden)
    idx = cb.index(srcs)
    corpus, host = cb.Corpus(idx, ctx), cb.Corpus(idx, ctx, memory="host")
    rng = np.random.default_rng(11)
    files, offsets, lengths = [], [], []
    for fi, f in enumerate(idx.files):
        N, st = f.length, f.starts.tolist()
        for o, ln in ((0, 1), (N - 1, -1), (N, -1), (N, 5), (0, -1), (st[-1], 3), (st[min(2, len(st) - 1)], 4097),
                      (int(rng.integers(0, N)), int(rng.integers(1, 3000))), (max(0, N - 2), 1)):
            files.append(fi)
            offsets.append(o)
            lengths.append(ln)
    perm = rng.permutation(len(files))
    files, offsets, lengths = ([x[p] for p in perm] for x in (files, offsets, lengths))
    T = sum((min(f.length, 10 ** 9) + 3) & ~3 for f in idx.files) * 3
    batch, hbatch = corpus.packed(len(files), T, dtype=dtype), host.packed(len(files), T, dtype=dtype)
    check_call(batch, idx, srcs, files, offsets, lengths, ctx, host=hbatch)
    # each excerpt also against load_crops() of it alone
    out, starts, lens = batch(files, offsets, lengths)
    for b in range(0, len(files), 3):
        n = int(lens[b])
        if n:
            exp, _ = cb.load_crops(idx, [files[b]], [offsets[b]], n, dtype=dtype, ctx=ctx)
            s = int(starts[b])
            c = exp.shape[1]
            assert torch.equal(bits(out[:c, s:s + n]), bits(exp[0])) and not bits(out[c:, s:s + n]).any(), b


# --------------------------------------------------------------------------- 2. capacity, zero-fill, invalid requests

@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_capacity_and_refused_suffix(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    srcs = files_1_2_4(golden)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    # an exact fit: 3 excerpts whose last one ends at T
    n0, n1, n2 = 1001, 4096, 777
    T = ((n0 + 3) & ~3) + ((n1 + 3) & ~3) + n2
    batch = corpus.packed(6, T, dtype=dtype)
    files, offsets = [0, 1, 2], [5, 0, 100]
    out = check_call(batch, idx, srcs, files, offsets, [n0, n1, n2], ctx)
    # one sample over: the last one and every later one are refused
    check_call(batch, idx, srcs, files + [3, 0], offsets + [0, 0], [n0, n1, n2 + 1, 1, 4], ctx)
    with pytest.raises(ValueError, match=f"excerpt 2: needs columns \\[{T - n2}, {T + 1}\\)"):
        batch(files, offsets, [n0, n1, n2 + 1])
    # count 0, then count == max_excerpts
    out, starts, lengths = batch([], check=True)
    assert starts.numel() == 0 and not bits(out).any()
    check_call(batch, idx, srcs, [0] * 6, [0, 10, 20, 30, 40, 50], [100] * 6, ctx)
    with pytest.raises(ValueError):
        batch([0] * 7)


@gpu
def test_long_call_then_short_call_equals_fresh_batch(ctx, golden):
    import torch
    srcs = files_1_2_4(golden)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    T = 300_000
    batch = corpus.packed(8, T, dtype=torch.int32)
    batch(list(range(7)), check=False)  # whole files, as many as fit in T
    short = ([2, 0, 3], [7, 0, 1], [50, 9, 3000])
    out, _, _ = batch(*short)
    fresh, _, _ = corpus.packed(8, T, dtype=torch.int32)(*short)
    assert torch.equal(out, fresh)
    check_call(batch, idx, srcs, *short, ctx)


@gpu
def test_invalid_requests(ctx, golden):
    import torch
    srcs = files_1_2_4(golden)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    files, offsets, lengths = [0, 1, 7, 2, 0, 3, 1, 2, 1 << 32], [0, 5, 0, 0, -1, 0, idx[1].length + 1, 0, 0], \
        [100, 200, 5, 0, 5, -2, 3, 50, 1]
    bad = [2, 3, 4, 5, 6, 8]
    batch = corpus.packed(len(files), 100_000, dtype=torch.float32)
    batch([0] * len(files), check=False)  # whole files first: what the short call leaves must be zeroed
    out, starts, lens = batch(files, offsets, lengths, check=False)
    st = batch.status.cpu().tolist()
    assert [b for b in range(len(files)) if st[b]] == bad and all(st[b] == 90 for b in bad)
    assert lens.cpu().tolist() == [100, 200, 0, 0, 0, 0, 0, 50, 0]
    assert starts.cpu().tolist()[:3] == [0, 100, 300] and int(starts[7]) == 300
    valid = [b for b in range(len(files)) if b not in bad]
    exp, s_exp, _ = expected(idx, srcs, [files[b] for b in valid], [offsets[b] for b in valid],
                             [lengths[b] for b in valid], 100_000, torch.float32, ctx)
    assert torch.equal(bits(out), bits(exp))
    with pytest.raises(ValueError, match="excerpt 2: file index 7 out of range"):
        batch(files, offsets, lengths)
    with pytest.raises(ValueError, match="excerpt 0: length 0"):
        batch([0], [0], [0])
    with pytest.raises(TypeError):
        batch(torch.zeros(3))


def check_damaged(ctx, idx, files, offsets, lengths, dtype):
    """Each excerpt's status against load_crops() of it alone, the raise of the whole call against what that implies,
    and a host-corpus batch against the device-corpus one."""
    import torch
    corpus, host = cb.Corpus(idx, ctx), cb.Corpus(idx, ctx, memory="host")
    B = max(len(files), len(idx))
    T = max(sum((idx[f].length + 3) & ~3 for f in files), sum((f.length + 3) & ~3 for f in idx.files))
    batch, hbatch = corpus.packed(B, T, dtype=dtype), host.packed(B, T, dtype=dtype)
    hbatch(list(range(len(idx))), check=False)  # long spans first
    out, starts, lens = batch(files, offsets, lengths, check=False)
    ho, _, _ = hbatch(files, offsets, lengths, check=False)
    st = batch.status.cpu().tolist()
    assert hbatch.status.cpu().tolist() == st and torch.equal(hbatch._error, batch._error)
    first = None
    for b, (f, o, ln) in enumerate(zip(files, offsets, lengths)):
        n = int(lens[b])
        e = raised(idx, [f], [o], n, dtype, ctx) if n else None
        assert st[b] == (e.status if e else 0), (b, f, o)
        if e and first is None:
            first = (b, e)
        if not e and n:
            exp, _ = cb.load_crops(idx, [f], [o], n, dtype=dtype, ctx=ctx)
            s = int(starts[b])
            c = exp.shape[1]
            assert torch.equal(bits(out[:c, s:s + n]), bits(exp[0])) and torch.equal(bits(ho[:c, s:s + n]), bits(exp[0]))
    if first is None:
        batch(files, offsets, lengths)
    else:  # the excerpt the error word names (frame failures before trailing bytes, each in excerpt order)
        with pytest.raises(cb.Error) as got:
            batch(files, offsets, lengths)
        b = (int(batch._error.item()) >> 32) & ((1 << 30) - 1)
        assert st[b] != 0 and got.value == raised(idx, [files[b]], [offsets[b]], int(lens[b]), dtype, ctx)
        assert str(got.value).endswith(f"(file {files[b]}, excerpt {b})") and b >= first[0]
    return st


@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_damaged_files(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    idx = damaged_index(golden)
    s0 = int(idx[0].starts[16])
    st = check_damaged(ctx, idx, [3, 0, 1, 2, 0], [0, 0, 0, 0, s0 + 10], [-1, 3000, -1, -1, 100], dtype)
    assert st[0] == st[1] == 0 and st[2] == 23 and st[3] != 0 and st[4] != 0
    check_damaged(ctx, idx, [3, 2], [0, idx[2].length - 100], [-1, -1], dtype)


@gpu
def test_corruption_corpus(ctx):
    import torch
    data, offsets, lengths = corruption_corpus()
    descs, _ = cb.descs_from_offsets(data, offsets, lengths)
    files = []
    for i in range(0, descs.size, 4):
        o, n = int(offsets[i]), int(lengths[i])
        d = descs[i:i + 1].copy()
        d["byte_offset"], d["out_offset"] = 0, 0
        info = cb.StreamInfo(576, 576, None, None, 44100, int(d["n_channels"][0]), int(d["bits_per_sample"][0]), None,
                             bytes(16))
        files.append(cb.IndexedFile(data[o:o + n].copy(), info, d, cb.frame_starts(d), int(d["block_size"][0]), False))
    idx = cb.FlacIndex(files)
    fs = list(range(len(files)))
    st = check_damaged(ctx, idx, fs, [min(i % 5 * 100, files[i].length) for i in fs], [-1] * len(fs), torch.int32)
    assert len(set(st)) >= 4, sorted(set(st))


# --------------------------------------------------------------------------- 3. device-drawn requests, launches, refusals

@gpu
def test_device_drawn_requests_without_sync(ctx, golden):
    import torch
    srcs = files_1_2_4(golden)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    lengths_dev = torch.tensor([f.length for f in idx.files], device="cuda")
    a, b = corpus.packed(12, 150_000, dtype=torch.float32), corpus.packed(5, 40_000, dtype=torch.int32)
    gen = torch.Generator(device="cuda").manual_seed(3)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(3):
            for batch in (a, b):
                fi = torch.randint(0, len(idx), (batch.max_excerpts - it,), device="cuda", generator=gen)
                off = (torch.rand(fi.numel(), device="cuda", generator=gen) * (lengths_dev[fi] + 1)).long()
                off = torch.minimum(off, lengths_dev[fi])
                ln = torch.randint(-1, 20000, (fi.numel(),), device="cuda", generator=gen)
                ln = torch.where(ln == 0, torch.ones_like(ln), ln)
                out, starts, lengths = batch(fi, off, ln, check=False)
                draws.append((batch, fi, off, ln, out.clone(), starts.clone(), lengths.clone(), batch.status.clone()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for batch, fi, off, ln, out, starts, lengths, status in draws:
        exp, s_exp, l_exp = expected(idx, srcs, fi.tolist(), off.tolist(), ln.tolist(), batch.max_samples, batch.dtype, ctx)
        assert starts.cpu().tolist() == s_exp
        assert lengths.cpu().tolist() == [x if x is not None else 0 for x in l_exp]
        assert status.cpu().tolist() == [0 if x is not None else 90 for x in l_exp]
        assert torch.equal(bits(out), bits(exp))


@gpu
def test_launch_counts(ctx, golden):
    """A packed batch launches what a crop batch of the same corpus does; one kernel more over a host corpus."""
    import torch
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)

    def per_call(batch, *args):
        batch(*args, check=False)
        n0 = ctx.launch_count
        batch(*args, check=False)
        return ctx.launch_count - n0

    crops = per_call(dev.crops(4, 5000, dtype=torch.float32), [0, 1, 2, 3], [0, 0, 0, 0])
    packed = per_call(dev.packed(7, 100_000, dtype=torch.float32), list(range(7)))
    hpacked = per_call(host.packed(7, 100_000, dtype=torch.float32), list(range(7)))
    assert packed == crops and hpacked == packed + 1, (crops, packed, hpacked)


@gpu
def test_refusals(ctx):
    import torch
    L = ctx._L
    data = flac_of(synth.workload_config("c2", 8))
    f = cb.index(data)[0]
    wide = f.descs.copy()
    wide["bits_per_sample"][5] = 25
    ff = np.array([0, 4, 8], np.uint32)
    h = C.c_void_p()
    assert L.clx_corpus_create(ctx._h, data.ctypes.data, data.size, wide.ctypes.data, wide.size, ff.ctypes.data, 2,
                               C.byref(h)) == 0
    b = C.c_void_p()
    for args in ((4, 100, cb.OUT_CHANNELS_F32), (0, 100, cb.OUT_CHANNELS_I32), (4, 0, cb.OUT_CHANNELS_I32),
                 (1 << 30, 100, cb.OUT_CHANNELS_I32), (4, 1 << 62, cb.OUT_CHANNELS_I32), (4, 100, cb.OUT_PLANAR_I32),
                 (4, 100, cb.OUT_INTERLEAVED_I16), (4, 100, 6)):
        assert L.clx_batch_create_packed(ctx._h, h, *args, C.byref(b)) == 90, args
    assert L.clx_batch_create_packed(ctx._h, h, 4, 100, cb.OUT_CHANNELS_I32, C.byref(b)) == 0
    assert L.clx_batch_packed_stride(b) == 100 + 100 and L.clx_batch_crop_requests(b) is None
    assert L.clx_batch_packed_stride(None) == 0
    assert L.clx_corpus_destroy(ctx._h, h) == 90  # a live packed batch
    L.clx_batch_destroy(ctx._h, b)
    assert L.clx_corpus_destroy(ctx._h, h) == 0
    corpus = cb.Corpus(cb.index(data), ctx)
    with pytest.raises(ValueError):
        corpus.packed(0, 10)
    with pytest.raises(ValueError):
        corpus.packed(2, 10, dtype=torch.int16)
    batch = corpus.packed(2, 10, dtype=torch.int32)
    with pytest.raises(cb.Error) as e:
        corpus.close()
    assert e.value.status == 90
    del batch
    gc.collect()
    corpus.close()
