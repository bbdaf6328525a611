"""Host-resident corpora: Corpus(memory="host") and the crop batches over it (-m gpu, except the CPU tests at the end).

A host corpus keeps its compressed bytes in pinned host memory; each call of a crop batch gathers the selected crops'
spans of frames into a device staging buffer before the decode.  Every call is compared bit for bit with a crop batch
of a device corpus of the same index (out, lengths, status and the error word) and with load_crops().  The staging
buffer keeps bytes of earlier calls after each span, so calls whose spans are short follow calls whose spans are long.
"""
import ctypes as C

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from tests.test_gpu_batch_out import corruption_corpus
from tests.test_gpu_corpus import (bits, blocks_desc, check_exact, damaged_index, files_1_2_4, flac_of, raised,
                                   requests_of)

gpu = pytest.mark.gpu


def call(batch, files, offsets):
    """One unchecked call; clones of what it left: out (as int32 bits), lengths, status, the error word."""
    out, lengths = batch(files, offsets, check=False)
    return bits(out).clone(), lengths.clone(), batch.status.clone(), batch._error.clone()


def check_same(host, dev, files, offsets):
    """The host-corpus batch and the device-corpus batch on the same requests: the same lengths, statuses and error
    word, and the same rows for every crop that did not fail (a failed crop's rows are unspecified)."""
    import torch
    ho, hl, hs, he = call(host, files, offsets)
    do, dl, ds, de = call(dev, files, offsets)
    assert torch.equal(hl, dl) and torch.equal(hs, ds) and torch.equal(he, de)
    ok = (hs == 0).nonzero().flatten()
    assert torch.equal(ho[ok], do[ok]), torch.nonzero(ho[ok] != do[ok])[:4].tolist()
    return hs.cpu().tolist()


def span_starts(corpus, files, offsets, L):
    """The corpus byte offset of each request's first planned frame (None for a crop without frames)."""
    out = []
    for fi, o in zip(files, offsets):
        f = corpus.index[fi]
        idx, _, _ = cb.plan_range(f.descs, o, min(o + L, f.length), starts=f.starts)
        out.append(int(corpus.descs["byte_offset"][int(corpus.file_frames[fi]) + int(idx[0])]) if idx.size else None)
    return out


# --------------------------------------------------------------------------- 1. against device corpora and load_crops()

@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_host_crops_match_device_crops_and_load_crops(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    files, offsets = requests_of(idx)
    B = len(files)
    rng = np.random.default_rng(9)
    longest = max(f.length for f in idx.files)
    for L in (1, 7, 37, 1000, 3 * 4096 + 5, longest + 3):
        hb, db = host.crops(B, L, dtype=dtype), dev.crops(B, L, dtype=dtype)
        assert hb.out.shape == (B, 4, L) and hb.out.dtype == dtype
        # long spans first (every crop from its file's start), then the mixed requests: short spans on stale bytes
        long_f = [b % len(idx) for b in range(B)]
        check_same(hb, db, long_f, [0] * B)
        assert check_same(hb, db, files, offsets) == [0] * B
        out, lengths = hb(files, offsets)
        check_exact(idx, out, lengths, files, offsets, L, dtype, ctx)
        perm = rng.permutation(B)
        f2, o2 = [files[p] for p in perm], [offsets[p] for p in perm]
        check_same(hb, db, torch.tensor(f2), torch.tensor(o2))
        out, lengths = hb(f2, o2)
        check_exact(idx, out, lengths, f2, o2, L, dtype, ctx)
        # every crop at its file's end (no frames, nothing gathered), then the mixed requests again
        o3 = [idx[f].length for f in long_f]
        out, lengths = hb(long_f, o3)
        assert not bits(out).any() and not lengths.any()
        check_same(hb, db, files, offsets)
        del hb, db


@gpu
def test_span_starts_cover_every_residue_mod_16(ctx, golden):
    """Requests whose spans start at all 16 residues mod 16 (so every head and tail length of the vector copy)."""
    import torch
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    L = 2500
    files, offsets = [], []
    for fi, f in enumerate(idx.files):
        for s in f.starts.tolist():
            files.append(fi)
            offsets.append(min(int(s) + 3, f.length))
    starts = span_starts(host, files, offsets, L)
    assert {s % 16 for s in starts if s is not None} == set(range(16))
    hb, db = host.crops(len(files), L, dtype=torch.int32), dev.crops(len(files), L, dtype=torch.int32)
    check_same(hb, db, [0] * len(files), [0] * len(files))
    check_same(hb, db, files, offsets)
    out, lengths = hb(files, offsets)
    check_exact(idx, out, lengths, files, offsets, L, torch.int32, ctx)


@gpu
def test_device_drawn_requests_without_sync(ctx, golden):
    """Requests drawn with torch.randint on the GPU, check=False under sync debug mode "error"; two crop batches of
    one host corpus interleaved."""
    import torch
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    lengths_dev = torch.tensor([f.length for f in idx.files], device="cuda")
    a, b = host.crops(40, 5000, dtype=torch.float32), host.crops(24, 333, dtype=torch.int32)
    gen = torch.Generator(device="cuda").manual_seed(3)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(3):
            for batch in (a, b):
                fi = torch.randint(0, len(idx), (batch.batch,), device="cuda", generator=gen)
                off = (torch.rand(batch.batch, device="cuda", generator=gen) * (lengths_dev[fi] + 1)).long()
                off = torch.minimum(off, lengths_dev[fi])
                out, lengths = batch(fi, off, check=False)
                draws.append((batch, fi, off, out.clone(), lengths.clone(), batch.status.clone()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    dev_batches = {id(a): dev.crops(40, 5000, dtype=torch.float32), id(b): dev.crops(24, 333, dtype=torch.int32)}
    for batch, fi, off, out, lengths, status in draws:
        assert not status.any()
        check_exact(idx, out, lengths, fi.tolist(), off.tolist(), batch.num_frames, batch.dtype, ctx)
        do, dl = dev_batches[id(batch)](fi, off)
        assert torch.equal(bits(out), bits(do)) and torch.equal(lengths, dl)


@gpu
def test_invalid_requests(ctx, golden):
    import torch
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    files, offsets = requests_of(idx)
    bad = {3: (len(idx), 0), 7: (-1, 0), 11: (0, -1), 12: (1, idx[1].length + 1), 20: (2, -(1 << 40)),
           21: (1 << 32, 0)}
    for b, (f, o) in bad.items():
        files[b], offsets[b] = f, o
    valid = [b for b in range(len(files)) if b not in bad]
    hb, db = host.crops(len(files), 4100, dtype=torch.float32), dev.crops(len(files), 4100, dtype=torch.float32)
    check_same(hb, db, [0] * len(files), [0] * len(files))  # long crops first: the bad crops' rows must then be zeroed
    st = check_same(hb, db, files, offsets)
    assert [b for b in range(len(files)) if st[b] != 0] == sorted(bad) and all(st[b] == 90 for b in bad)
    out, lengths = hb(files, offsets, check=False)
    assert not bits(out[sorted(bad)]).any() and not lengths[sorted(bad)].any()
    check_exact(idx, out, lengths, files, offsets, 4100, torch.float32, ctx, valid=valid)
    with pytest.raises(ValueError) as e:
        hb(files, offsets)
    with pytest.raises(ValueError) as e_lc:
        cb.load_crops(idx, files, offsets, 4100, ctx=ctx)
    assert str(e.value) == str(e_lc.value) == f"crop 3: file index {len(idx)} out of range"
    files[3], offsets[3] = 0, 0
    with pytest.raises(ValueError) as e:
        hb(files, offsets)
    with pytest.raises(ValueError) as e_lc:
        cb.load_crops(idx, files, offsets, 4100, ctx=ctx)
    assert str(e.value) == str(e_lc.value)


# --------------------------------------------------------------------------- 2. damaged files

def check_damaged_host(ctx, idx, files, offsets, L, dtype):
    """Each crop's status against load_crops() of it alone, its rows against load_crops() when it decodes, the whole
    batch's raise against load_crops()', and everything against a device-corpus batch; after a call of long spans."""
    import torch
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    hb, db = host.crops(len(files), L, dtype=dtype), dev.crops(len(files), L, dtype=dtype)
    check_same(hb, db, [b % len(idx) for b in range(len(files))], [0] * len(files))
    st = check_same(hb, db, files, offsets)
    out, _ = hb(files, offsets, check=False)
    for b, (f, o) in enumerate(zip(files, offsets)):
        e = raised(idx, [f], [o], L, dtype, ctx)
        assert st[b] == (e.status if e else 0), (b, f, o)
        if not e:
            exp, _ = cb.load_crops(idx, [f], [o], L, dtype=dtype, ctx=ctx)
            assert torch.equal(bits(out[b, :exp.shape[1]]), bits(exp[0])), b
    e_lc = raised(idx, files, offsets, L, dtype, ctx)
    if e_lc is None:
        hb(files, offsets)
    else:
        with pytest.raises(cb.Error) as e:
            hb(files, offsets)
        assert e.value == e_lc and str(e.value) == str(e_lc)
    return st


@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_damaged_files(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    idx = damaged_index(golden)
    s0, bs = int(idx[0].starts[16]), 4096
    L = 3000
    files = [3, 0, 0, 1, 2, 2, 0, 3, 1]
    offsets = [0, 0, s0 + bs - 10, int(idx[1].starts[9]) + 5, 0, idx[2].length - 100, s0 + 10, 50, 0]
    st = check_damaged_host(ctx, idx, files, offsets, L, dtype)
    assert st[2] != 0 and st[6] != 0 and st[3] == 23 and st[5] != 0 and st[0] == st[1] == st[4] == st[8] == 0
    # an unconfirmed last frame followed by trailing bytes: the verdict is what is raised
    check_damaged_host(ctx, idx, [3, 2, 1, 2], [0, idx[2].length - 100, 0, 0], L, dtype)
    check_damaged_host(ctx, idx, [2, 0], [idx[2].length - 1, s0], L, dtype)


@gpu
def test_corruption_corpus(ctx):
    """Each frame of the corruption corpus as a file of its own, its end unconfirmed."""
    import torch
    data, offsets, lengths = corruption_corpus()
    descs, _ = cb.descs_from_offsets(data, offsets, lengths)
    files = []
    for i in range(0, descs.size, 4):
        o, n = int(offsets[i]), int(lengths[i])
        d = descs[i:i + 1].copy()
        d["byte_offset"], d["out_offset"] = 0, 0
        nch = int(d["n_channels"][0])
        info = cb.StreamInfo(576, 576, None, None, 44100, nch, int(d["bits_per_sample"][0]), None, bytes(16))
        files.append(cb.IndexedFile(data[o:o + n].copy(), info, d, cb.frame_starts(d), int(d["block_size"][0]), False))
    idx = cb.FlacIndex(files)
    fs = list(range(len(files)))
    st = check_damaged_host(ctx, idx, fs, [min(i % 5 * 100, files[i].length) for i in fs], 300, torch.int32)
    assert len(set(st)) >= 4, sorted(set(st))


# --------------------------------------------------------------------------- 3. full size, memory, launches, refusals

@gpu
def test_full_size_workload(ctx):
    """256 crops of 176 400 samples of C2-shaped files, f32, against load_crops() and a device corpus."""
    import torch
    srcs = [flac_of(synth.workload_config("c2", 300)), flac_of(synth.workload_config("c2", 250, seed=11))]
    idx = cb.index(srcs)
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    n = 176400
    rng = np.random.default_rng(4)
    files = rng.integers(0, 2, 256).tolist()
    offsets = [int(rng.integers(0, idx[f].length - n)) for f in files]
    hb, db = host.crops(256, n), dev.crops(256, n)
    assert check_same(hb, db, files, offsets) == [0] * 256
    out, lengths = hb(files, offsets)
    exp, elen = cb.load_crops(idx, files, offsets, n, ctx=ctx)
    assert torch.equal(lengths.cpu(), elen) and (elen == n).all()
    assert torch.equal(bits(out), bits(exp))


@gpu
def test_device_bytes(ctx, golden):
    """A host corpus holds only its frame index on the device, whatever its bytes; a device corpus holds its bytes."""
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    nf, nfiles = host.descs.size, len(idx)
    index_bytes = (nf + 1) * 40 + nf * 8 + (nfiles + 1) * 4 + nfiles * (8 + 4 + 4)
    assert host.device_bytes <= index_bytes + 64, (host.device_bytes, index_bytes)
    assert host.nbytes > 10 * index_bytes
    assert dev.device_bytes >= dev.nbytes + index_bytes
    # the same frame index over 1 MB more bytes: the host corpus's device memory does not change
    big = [np.concatenate([f.data, np.zeros(1 << 20, np.uint8)]) if i == 0 else f.data for i, f in enumerate(idx.files)]
    idx2 = cb.FlacIndex([cb.IndexedFile(d, f.info, f.descs, f.starts, f.length, f.end_confirmed)
                         for d, f in zip(big, idx.files)])
    host2 = cb.Corpus(idx2, ctx, memory="host")
    assert host2.nbytes == host.nbytes + (1 << 20) and host2.device_bytes == host.device_bytes


@gpu
def test_launch_counts(ctx, golden):
    """A crop batch of a host corpus launches exactly one kernel more per call than one of a device corpus."""
    import torch
    idx = cb.index(files_1_2_4(golden))
    host, dev = cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)
    files, offsets = requests_of(idx)
    counts = []
    for corpus in (host, dev):
        batch = corpus.crops(len(files), 5000, dtype=torch.float32)
        batch(files, offsets)
        n0 = ctx.launch_count
        batch(files, offsets)
        counts.append(ctx.launch_count - n0)
    assert counts[0] == counts[1] + 1, counts


def corpus_create_ex(c, data, descs, file_frames, flags):
    h = C.c_void_p()
    ff = np.asarray(file_frames, dtype=np.uint32)
    st = c._L.clx_corpus_create_ex(c._h, data.ctypes.data, data.size, descs.ctypes.data, descs.size, ff.ctypes.data,
                                   ff.size - 1, flags, C.byref(h))
    return st, h


@gpu
def test_refusals(ctx):
    import torch
    L = ctx._L
    data = flac_of(synth.workload_config("c2", 8))
    descs = cb.index(data)[0].descs
    for flags in (2, 3, 1 << 31):
        assert corpus_create_ex(ctx, data, descs, [0, 8], flags)[0] == 90, flags
    swapped = descs[[0, 2, 1, 3, 4, 5, 6, 7]].copy()  # out of byte order: refused for a host corpus only
    assert corpus_create_ex(ctx, data, swapped, [0, 8], 1)[0] == 90
    st, h = corpus_create_ex(ctx, data, swapped, [0, 8], 0)
    assert st == 0 and L.clx_corpus_destroy(ctx._h, h) == 0
    st, h = corpus_create_ex(ctx, data, swapped, [0, 2, 8], 1)  # ... and fine across files
    assert st == 0 and L.clx_corpus_destroy(ctx._h, h) == 0
    st, h = corpus_create_ex(ctx, data, descs, [0, 4, 8], 1)
    assert st == 0
    b = C.c_void_p()
    assert L.clx_batch_create_crops(ctx._h, h, 4, 100, cb.OUT_CHANNELS_I32, C.byref(b)) == 0
    assert L.clx_corpus_destroy(ctx._h, h) == 90  # a live batch
    L.clx_batch_destroy(ctx._h, b)
    assert L.clx_corpus_destroy(ctx._h, h) == 0
    corpus = cb.Corpus(cb.index(data), ctx, memory="host")
    batch = corpus.crops(2, 10, dtype=torch.int32)
    with pytest.raises(cb.Error) as e:
        corpus.close()
    assert e.value.status == 90
    del batch
    import gc
    gc.collect()
    corpus.close()


# --------------------------------------------------------------------------- CPU: the byte bound, exports, arguments

def with_bytes(d, rng):
    """Descriptors with random frame lengths, laid out back to back from a random start."""
    d = d.copy()
    d["byte_len"] = rng.integers(11, 3 * 4096, d.size)
    d["byte_offset"] = int(rng.integers(0, 100)) + np.concatenate([[0], np.cumsum(d["byte_len"][:-1].astype(np.int64))])
    return d


def bytes_bound_of(group, L):
    descs = np.concatenate(group) if group else np.zeros(0, dtype=cb.DESC_DTYPE)
    ff = np.concatenate([[0], np.cumsum([d.size for d in group])]).astype(np.uint32)
    return int(_lib.load().clx_crop_bytes_bound(descs.ctypes.data, descs.size, ff.ctypes.data, len(group), L))


def frames_bound_of(group, L):
    descs = np.concatenate(group)
    ff = np.concatenate([[0], np.cumsum([d.size for d in group])]).astype(np.uint32)
    return int(_lib.load().clx_crop_frames_bound(descs.ctypes.data, descs.size, ff.ctypes.data, len(group), L))


def real_spans(d, L):
    """The bytes from the first to the end of the last frame plan_range() selects, for num_frames = L at every offset
    of the file (vectorised over the offsets; plan_range itself on a sample of them)."""
    starts = cb.frame_starts(d)
    bs = d["block_size"].astype(np.int64)
    N = int(bs.sum())
    lo = np.arange(N + 1, dtype=np.int64)
    hi = np.minimum(lo + L, N)
    i0 = np.searchsorted(starts + bs, lo, side="right")
    i1 = np.where(hi > lo, np.searchsorted(starts, hi, side="left"), i0)
    has = i1 > i0
    off = d["byte_offset"].astype(np.int64)
    end = off + d["byte_len"].astype(np.int64)
    span = np.where(has, end[np.maximum(i1 - 1, 0)] - off[np.minimum(i0, d.size - 1)], 0)
    for o in np.random.default_rng(L).integers(0, N + 1, 20):
        idx, _, _ = cb.plan_range(d, int(o), min(int(o) + L, N))
        assert span[o] == (int(end[idx[-1]] - off[idx[0]]) if idx.size else 0)
    return int(span.max())


def window_max(group, S):
    """The largest end of frame min(f + S, file's frames) - 1 minus the start of frame f, over every frame f."""
    most = 0
    for d in group:
        off = d["byte_offset"].astype(np.int64)
        end = off + d["byte_len"].astype(np.int64)
        last = np.minimum(np.arange(d.size) + S, d.size) - 1
        if d.size:
            most = max(most, int((end[last] - off).max()))
    return most


def test_crop_bytes_bound_brute_force(golden):
    idx = cb.index([golden[f"{n}__bytes"] for n in ("pop", "short", "wasted_bits")])
    rng = np.random.default_rng(1)
    synthetic = [with_bytes(d, rng) for d in (
        blocks_desc([4096] * 20 + [1001]),
        blocks_desc(rng.integers(16, 65536, 12).tolist() + [7]),
        blocks_desc([16] * 50 + [65535, 16, 3]),
        blocks_desc(rng.integers(16, 300, 40).tolist()),
        blocks_desc([5000]),
    )]
    golden_group = [f.descs for f in idx.files]
    for group in (golden_group, synthetic, synthetic[:2], [synthetic[4]], synthetic[2:3]):
        for L in (1, 2, 3, 15, 16, 17, 100, 4095, 4096, 4097, 8194, 70000, 10 ** 6):
            got = bytes_bound_of(group, L)
            assert got == window_max(group, frames_bound_of(group, L)), L
            assert got >= max(real_spans(d, L) for d in group), L
    assert bytes_bound_of(synthetic[:1], 0) == 0
    d = synthetic[0]
    for ff, n in (([0, 5, 3, 21], 3), ([0, 20], 1)):  # not monotone; not ending at n_frames
        ff = np.array(ff, np.uint32)
        assert _lib.load().clx_crop_bytes_bound(d.ctypes.data, d.size, ff.ctypes.data, n, 100) == 0


def test_host_corpus_entry_points_are_exported():
    lib = C.CDLL(_lib.load()._name)
    for name in ("clx_corpus_create_ex", "clx_corpus_device_bytes", "clx_crop_bytes_bound"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS, name
    assert _lib.CORPUS_HOST == 1


def test_corpus_memory_argument(golden):
    idx = cb.index(golden["short__bytes"])
    for memory in ("HOST", "pinned", None, ""):
        with pytest.raises(ValueError):
            cb.Corpus(idx, memory=memory)
