"""Device-resident corpora and crop batches: Corpus, CropBatch and the C ABI under them (-m gpu, except the CPU tests at
the end).

A crop batch plans each call's frames, windows and columns on the device.  Every valid request is compared bit for bit
with load_crops() on the same index, which gathers and plans on the host: the tensor (the batch's rows beyond the
chosen files' largest channel count must read 0) and the lengths.  Statuses and raises are compared with what
load_crops() raises for the same requests.
"""
import ctypes as C
import hashlib

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from tests.test_gpu_batch_out import corruption_corpus

gpu = pytest.mark.gpu


def flac_of(cfg):
    b = synth.generate(cfg)
    return np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy()


def c4ch_config():  # 4 channels, 2048-sample blocks
    cfg = synth.workload_config("c2", 12)
    cfg.n_channels, cfg.block_size, cfg.stereo_mode = 4, 2048, synth.INDEPENDENT
    return cfg


def variable_config():  # variable blocking: 1152-sample blocks, every third one 37 samples
    return synth.SynthConfig(seed=77, n_frames=14, block_size=1152, tail_block_size=37, frames_per_file=3,
                             n_channels=1, bps=16, variable_blocking=1, type_mask=synth.TYPE_FIXED | synth.TYPE_LPC,
                             lpc_min_order=1, lpc_max_order=8, rice_mode=-1)


_files = {}


def files_1_2_4(golden):
    """Files of 1, 2 and 4 channels, fixed and variable block sizes (C = 4)."""
    if "srcs" not in _files:
        _files["srcs"] = [flac_of(synth.workload_config("c2", 30)), flac_of(synth.workload_config("c4", 23)),
                          flac_of(c4ch_config()), flac_of(variable_config()),
                          golden["pop__bytes"], golden["short__bytes"], golden["wasted_bits__bytes"]]
    return _files["srcs"]


def bits(t):
    import torch
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def check_exact(idx, out, lengths, files, offsets, L, dtype, ctx, valid=None):
    """out / lengths of a crop batch against load_crops() of the valid requests."""
    import torch
    valid = list(range(len(files))) if valid is None else valid
    exp, elen = cb.load_crops(idx, [files[b] for b in valid], [offsets[b] for b in valid], L, dtype=dtype, ctx=ctx)
    got = bits(out[valid])
    C_ = exp.shape[1]
    assert torch.equal(lengths[valid].cpu(), elen), (L,)
    assert torch.equal(got[:, :C_], bits(exp)), (L, torch.nonzero(got[:, :C_] != bits(exp))[:4].tolist())
    assert not got[:, C_:].any(), L


def requests_of(idx):
    """Offsets at frame boundaries, inside frames, 0, length - 1 and length, for every file."""
    files, offsets = [], []
    rng = np.random.default_rng(5)
    for fi, f in enumerate(idx.files):
        N, st = f.length, f.starts.tolist()
        cand = {0, N, max(0, N - 1), max(0, N - 3)}
        if len(st) > 2:
            cand |= {st[1], st[2] - 1, st[-1], st[-1] - 1, st[1] + 5}
        cand |= set(int(x) for x in rng.integers(0, N + 1, 3))
        for o in sorted(cand):
            files.append(fi)
            offsets.append(int(o))
    return files, offsets


# --------------------------------------------------------------------------- 1. against load_crops()

@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_crops_match_load_crops(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    idx = cb.index(files_1_2_4(golden))
    corpus = cb.Corpus(idx, ctx)
    assert corpus.channels == 4
    files, offsets = requests_of(idx)
    B = len(files)
    rng = np.random.default_rng(9)
    longest = max(f.length for f in idx.files)
    for L in (1, 7, 37, 1000, 3 * 4096 + 5, longest + 3):
        batch = corpus.crops(B, L, dtype=dtype)
        assert batch.out.shape == (B, 4, L) and batch.out.dtype == dtype
        out, lengths = batch(files, offsets)
        check_exact(idx, out, lengths, files, offsets, L, dtype, ctx)
        # the same batch again: shuffled requests, then every crop at its file's end after long crops (nothing stale)
        perm = rng.permutation(B)
        f2, o2 = [files[p] for p in perm], [offsets[p] for p in perm]
        out, lengths = batch(torch.tensor(f2), torch.tensor(o2))
        check_exact(idx, out, lengths, f2, o2, L, dtype, ctx)
        f3 = [b % len(idx) for b in range(B)]
        o3 = [idx[f].length for f in f3]
        out, lengths = batch(f3, o3)
        assert not bits(out).any() and not lengths.any()
        out, lengths = batch(files, offsets)
        check_exact(idx, out, lengths, files, offsets, L, dtype, ctx)
        assert not batch.status.any()
    with pytest.raises(ValueError):
        batch(files[:-1], offsets[:-1])


@gpu
def test_device_drawn_requests_without_sync(ctx, golden):
    """Requests drawn with torch.randint on the GPU, check=False under sync debug mode "error"; two crop batches of
    one corpus interleaved."""
    import torch
    idx = cb.index(files_1_2_4(golden))
    corpus = cb.Corpus(idx, ctx)
    lengths_dev = torch.tensor([f.length for f in idx.files], device="cuda")
    a, b = corpus.crops(40, 5000, dtype=torch.float32), corpus.crops(24, 333, dtype=torch.int32)
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
    for batch, fi, off, out, lengths, status in draws:
        assert not status.any()
        check_exact(idx, out, lengths, fi.tolist(), off.tolist(), batch.num_frames, batch.dtype, ctx)


@gpu
def test_invalid_requests(ctx, golden):
    import torch
    idx = cb.index(files_1_2_4(golden))
    corpus = cb.Corpus(idx, ctx)
    files, offsets = requests_of(idx)
    bad = {3: (len(idx), 0), 7: (-1, 0), 11: (0, -1), 12: (1, idx[1].length + 1), 20: (2, -(1 << 40)),
           21: (1 << 32, 0)}
    for b, (f, o) in bad.items():
        files[b], offsets[b] = f, o
    valid = [b for b in range(len(files)) if b not in bad]
    batch = corpus.crops(len(files), 4100, dtype=torch.float32)
    batch([0] * len(files), [0] * len(files))  # long crops first: the bad crops' rows must then be zeroed
    out, lengths = batch(files, offsets, check=False)
    st = batch.status.cpu()
    assert [b for b in range(len(files)) if st[b] != 0] == sorted(bad) and (st[sorted(bad)] == 90).all()
    assert not bits(out[sorted(bad)]).any() and not lengths[sorted(bad)].any()
    check_exact(idx, out, lengths, files, offsets, 4100, torch.float32, ctx, valid=valid)
    with pytest.raises(ValueError) as e:
        batch(files, offsets)
    with pytest.raises(ValueError) as e_lc:
        cb.load_crops(idx, files, offsets, 4100, ctx=ctx)
    assert str(e.value) == str(e_lc.value) == f"crop 3: file index {len(idx)} out of range"
    with pytest.raises(TypeError):
        batch(torch.zeros(len(files)), offsets)


# --------------------------------------------------------------------------- 2. damaged files

def damaged_index(golden):
    """A file with one corrupted frame in the middle, one with a CRC-16 mismatch, one with garbage after an
    unconfirmed last frame, a clean one."""
    corrupt = flac_of(synth.workload_config("c4", 33))
    d = cb.index(corrupt)[0].descs[16]
    corrupt[int(d["byte_offset"]) + int(d["byte_len"]) // 2] ^= 0x10
    crc = flac_of(synth.workload_config("c2", 20))
    d = cb.index(crc)[0].descs[9]
    crc[int(d["byte_offset"]) + int(d["byte_len"]) - 3] ^= 0x01  # the last data byte before the CRC-16
    tail = np.concatenate([flac_of(synth.workload_config("c2", 6)), np.frombuffer(b"\xff\xf8junk!", np.uint8)])
    idx = cb.index([corrupt, crc, tail, golden["pop__bytes"]])
    assert not idx[2].end_confirmed
    return idx


def raised(idx, files, offsets, L, dtype, ctx):
    try:
        cb.load_crops(idx, files, offsets, L, dtype=dtype, ctx=ctx)
    except cb.Error as e:
        return e
    return None


def check_damaged(ctx, idx, files, offsets, L, dtype):
    import torch
    corpus = cb.Corpus(idx, ctx)
    batch = corpus.crops(len(files), L, dtype=dtype)
    out, lengths = batch(files, offsets, check=False)
    st = batch.status.cpu().tolist()
    for b, (f, o) in enumerate(zip(files, offsets)):
        e = raised(idx, [f], [o], L, dtype, ctx)
        assert st[b] == (e.status if e else 0), (b, f, o)
        if not e:
            exp, _ = cb.load_crops(idx, [f], [o], L, dtype=dtype, ctx=ctx)
            assert torch.equal(bits(out[b, :exp.shape[1]]), bits(exp[0])), b
    e_lc = raised(idx, files, offsets, L, dtype, ctx)
    if e_lc is None:
        batch(files, offsets)
    else:
        with pytest.raises(cb.Error) as e:
            batch(files, offsets)
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
    st = check_damaged(ctx, idx, files, offsets, L, dtype)
    assert st[2] != 0 and st[6] != 0 and st[3] == 23 and st[5] != 0 and st[0] == st[1] == st[4] == st[8] == 0
    # without the frame failures, the trailing-bytes verdict is what is raised
    check_damaged(ctx, idx, [3, 2, 1, 2], [0, idx[2].length - 100, 0, 0], L, dtype)
    # the crops alone (in load_crops' order: frame failures of any crop before trailing bytes)
    check_damaged(ctx, idx, [2, 0], [idx[2].length - 1, s0], L, dtype)


@gpu
def test_corruption_corpus(ctx):
    """Each frame of the corruption corpus as a file of its own, its end unconfirmed: every crop's status is what
    load_crops() raises for it alone, and the samples of every crop that decodes are load_crops()'."""
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
    st = check_damaged(ctx, idx, fs, [min(i % 5 * 100, files[i].length) for i in fs], 300, torch.int32)
    assert len(set(st)) >= 4, sorted(set(st))


# --------------------------------------------------------------------------- 3. MD5, full size, refusals

@gpu
def test_consecutive_crops_give_the_streaminfo_md5(golden):
    import torch
    for name in ("pop", "short", "wasted_bits"):
        data = golden[f"{name}__bytes"]
        si, _ = cb.open_stream(data)
        idx = cb.index(data)
        corpus = cb.Corpus(idx)
        offsets = list(range(0, idx[0].length, 1999))
        batch = corpus.crops(len(offsets), 1999, dtype=torch.int32)
        t, lengths = batch([0] * len(offsets), offsets)
        pcm = np.concatenate([t[b, :si.channels, :int(lengths[b])].cpu().numpy() for b in range(len(offsets))], axis=1)
        assert hashlib.md5(pcm.T.astype("<i2").tobytes()).digest() == si.md5sum, name


@gpu
def test_full_size_workload():
    """256 crops of 176 400 samples of C2-shaped files, f32, against load_crops()."""
    import torch
    srcs = [flac_of(synth.workload_config("c2", 300)), flac_of(synth.workload_config("c2", 250, seed=11))]
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx)
    n = 176400
    assert corpus.frames_bound(n) == 45
    rng = np.random.default_rng(4)
    files = rng.integers(0, 2, 256).tolist()
    offsets = [int(rng.integers(0, idx[f].length - n)) for f in files]
    batch = corpus.crops(256, n)
    out, lengths = batch(files, offsets)
    exp, elen = cb.load_crops(idx, files, offsets, n)
    assert torch.equal(lengths.cpu(), elen) and (elen == n).all()
    assert torch.equal(bits(out), bits(exp))


def corpus_create(c, data, descs, file_frames):
    h = C.c_void_p()
    ff = np.asarray(file_frames, dtype=np.uint32)
    st = c._L.clx_corpus_create(c._h, data.ctypes.data, data.size, descs.ctypes.data, descs.size, ff.ctypes.data,
                                ff.size - 1, C.byref(h))
    return st, h


@gpu
def test_refusals(ctx, golden):
    import torch
    L = ctx._L
    data = flac_of(synth.workload_config("c2", 8))
    f = cb.index(data)[0]
    descs = f.descs
    for ff in ([0, 5, 3, 8], [0, 4, 7], [0, 9], [1, 4, 9]):
        assert corpus_create(ctx, data, descs, ff)[0] == 90, ff
    bad = descs.copy()
    bad["byte_len"][2] = data.size  # beyond the bytes
    assert corpus_create(ctx, data, bad, [0, 8])[0] == 90
    bad = descs.copy()
    bad["n_channels"][3], bad["channel_assignment"][3] = 1, 0  # two channel counts in one file
    assert corpus_create(ctx, data, bad, [0, 8])[0] == 90
    st, h = corpus_create(ctx, data, bad, [0, 3, 4, 8])  # the odd frame as a file of its own
    assert st == 0 and L.clx_corpus_destroy(ctx._h, h) == 0
    wide = descs.copy()
    wide["bits_per_sample"][5] = 25
    st, h = corpus_create(ctx, data, wide, [0, 4, 8])
    assert st == 0
    b = C.c_void_p()
    assert L.clx_batch_create_crops(ctx._h, h, 4, 100, cb.OUT_CHANNELS_F32, C.byref(b)) == 90
    assert L.clx_batch_create_crops(ctx._h, h, 0, 100, cb.OUT_CHANNELS_I32, C.byref(b)) == 90
    assert L.clx_batch_create_crops(ctx._h, h, 4, 0, cb.OUT_CHANNELS_I32, C.byref(b)) == 90
    for mode in (cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I16, 6):
        assert L.clx_batch_create_crops(ctx._h, h, 4, 100, mode, C.byref(b)) == 90
    assert L.clx_batch_create_crops(ctx._h, h, 1 << 30, 100, cb.OUT_CHANNELS_I32, C.byref(b)) == 90
    assert L.clx_batch_create_crops(ctx._h, h, 4, 1 << 62, cb.OUT_CHANNELS_I32, C.byref(b)) == 90
    assert L.clx_batch_create_crops(ctx._h, h, 4, 100, cb.OUT_CHANNELS_I32, C.byref(b)) == 0
    assert L.clx_corpus_destroy(ctx._h, h) == 90  # a live batch
    L.clx_batch_destroy(ctx._h, b)
    assert L.clx_corpus_destroy(ctx._h, h) == 0
    # the Python layer: load_crops refuses F32 only for the frames a call selects; a crop batch for any frame
    idx = cb.index(data)
    corpus = cb.Corpus(idx, ctx)
    with pytest.raises(ValueError):
        corpus.crops(0, 10)
    batch = corpus.crops(2, 10, dtype=torch.int32)
    with pytest.raises(cb.Error) as e:
        corpus.close()
    assert e.value.status == 90
    del batch
    import gc
    gc.collect()
    corpus.close()


# --------------------------------------------------------------------------- CPU: the bound, the filler frame, exports

def bound_of(descs_per_file, L):
    descs = np.concatenate(descs_per_file) if descs_per_file else np.zeros(0, dtype=cb.DESC_DTYPE)
    ff = np.concatenate([[0], np.cumsum([d.size for d in descs_per_file])]).astype(np.uint32)
    return int(_lib.load().clx_crop_frames_bound(descs.ctypes.data, descs.size, ff.ctypes.data, len(descs_per_file), L))


def brute_force(descs, L):
    """The most frames plan_range() selects for num_frames = L over every offset of the file (vectorised over the
    offsets; plan_range itself on a sample of them)."""
    starts = cb.frame_starts(descs)
    bs = descs["block_size"].astype(np.int64)
    N = int(bs.sum())
    lo = np.arange(N + 1, dtype=np.int64)
    hi = np.minimum(lo + L, N)
    i0 = np.searchsorted(starts + bs, lo, side="right")
    i1 = np.where(hi > lo, np.searchsorted(starts, hi, side="left"), i0)
    count = np.maximum(i1 - i0, 0)
    for o in np.random.default_rng(L).integers(0, N + 1, 20):
        assert plan_count(descs, int(o), L) == count[o]
    return int(count.max())


def plan_count(descs, o, L):
    n = int(descs["block_size"].astype(np.int64).sum())
    return cb.plan_range(descs, o, min(o + L, n))[0].size


def blocks_desc(blocks):
    d = np.zeros(len(blocks), dtype=cb.DESC_DTYPE)
    d["block_size"], d["n_channels"] = blocks, 2
    return d


def test_crop_frames_bound_brute_force(golden):
    idx = cb.index([golden[f"{n}__bytes"] for n in ("pop", "short", "wasted_bits")])
    rng = np.random.default_rng(1)
    synthetic = [
        blocks_desc([4096] * 20 + [1001]),
        blocks_desc(rng.integers(16, 65536, 12).tolist() + [7]),
        blocks_desc([16] * 50 + [65535, 16, 3]),
        blocks_desc(rng.integers(16, 300, 40).tolist()),
        blocks_desc([5000]),
    ]
    for group in ([f.descs for f in idx.files], synthetic, synthetic[:2], [synthetic[4]], synthetic[2:3]):
        nonlast = [int(d["block_size"][:-1].min()) for d in group if d.size > 1]
        most = max(d.size for d in group)
        for L in (1, 2, 3, 15, 16, 17, 100, 4095, 4096, 4097, 8194, 70000, 10 ** 6):
            got = bound_of(group, L)
            exp = 1 if not nonlast or L == 1 else max(1, min((L - 2) // min(nonlast) + 2, most))
            assert got == exp, (L, got, exp)
            assert got >= max(brute_force(d, L) for d in group), L
    assert bound_of(synthetic[:1], 0) == 0
    d = synthetic[0]
    ff = np.array([0, 5, 3, 21], np.uint32)
    assert _lib.load().clx_crop_frames_bound(d.ctypes.data, d.size, ff.ctypes.data, 3, 100) == 0
    ff = np.array([0, 20], np.uint32)  # does not end at n_frames
    assert _lib.load().clx_crop_frames_bound(d.ctypes.data, d.size, ff.ctypes.data, 1, 100) == 0


def test_filler_frame_decodes_to_zeros():
    from oracle import oracle as O
    L = _lib.load()
    n = L.clx_crop_filler_frame(None, 0)
    buf = np.zeros(n, np.uint8)
    assert L.clx_crop_filler_frame(buf.ctypes.data, n) == n == 11
    st, d = cb.parse_frame_header(buf)
    assert st == 0 and d.block_size == 192 and d.n_channels == 1 and d.bits_per_sample == 16 and d.header_len == 6
    assert L.clx_crc8(buf.ctypes.data, 5) == buf[5]
    assert L.clx_crc16(buf.ctypes.data, n - 2) == (int(buf[-2]) << 8 | int(buf[-1]))
    fr = O.decode_frame(buf, verify_crc=True)
    assert fr.status == 0 and fr.samples.size == 192 and not fr.samples.any()
    dd, _, _, stop = cb.demux_frames(buf)
    assert dd.size == 1 and dd["byte_len"][0] == n and dd["flags"][0] & cb.FRAME_CRC16_VERIFIED and stop == cb.EOF


def test_corpus_entry_points_are_exported():
    lib = C.CDLL(_lib.load()._name)
    for name in ("clx_corpus_create", "clx_corpus_destroy", "clx_batch_create_crops", "clx_crop_frames_bound",
                 "clx_batch_crop_requests", "clx_batch_crop_status", "clx_batch_crop_lengths", "clx_batch_crop_error",
                 "clx_crop_filler_frame"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS, name
    for name in ("Corpus", "CropBatch"):
        assert name in cb.__all__
