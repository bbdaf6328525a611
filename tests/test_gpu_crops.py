"""Sample ranges of FLAC streams on the device: windowed channels-first batches, index(), load_crops() and
load(frame_offset, num_frames) (-m gpu, except the CPU tests at the end).

A windowed batch (clx_batch_create_windows) stores, for each frame, only samples [first, first + count) of each
channel c, on row `row + c`, from column out_offset on.  Everything is compared with the oracle's or the generator's
PCM cut and placed on the host, with the planar batch of the same frames, and with slices of load().
"""
import ctypes as C
import hashlib

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from tests import fastpath as F
from tests.test_gpu_batch_out import CASES, WRAPPING_16, corruption_corpus, oracle_of, resident, stream
from tests.test_gpu_channels import GOLDEN_AUDIO, NAMES, F32, I32, bits, channels_batch, columns, modes_for
from tests.test_gpu_launch_sequence import CONFIGS
from tests.test_gpu_mixed import PARTS

gpu = pytest.mark.gpu


def random_windows(descs, rows, kind, seed):
    """(windows, cols, stride) of a random layout: every frame on a random row base, columns one after the other
    (odd, or 4-aligned, with a stride of the same kind), windows that clip both ends, hold one sample, start at the
    block's last sample, clip one end, or are full."""
    rng = np.random.default_rng(seed)
    w = np.zeros(descs.size, dtype=cb.WINDOW_DTYPE)
    cols = np.zeros(descs.size, np.uint64)
    at = 3 if kind == "odd" else 0
    for i, d in enumerate(descs):
        bs, nch = int(d["block_size"]), int(d["n_channels"])
        pick = i % 6
        if pick == 0 and bs > 2:  # both ends
            first = int(rng.integers(1, bs - 1))
            count = int(rng.integers(1, bs - first))
        elif pick == 1:
            first, count = int(rng.integers(0, bs)), 1
        elif pick == 2:
            first, count = bs - 1, 1
        elif pick == 3:  # the start only
            first = int(rng.integers(0, bs))
            count = bs - first
        elif pick == 4:  # the end only
            first, count = 0, int(rng.integers(1, bs + 1))
        else:
            first, count = 0, bs
        w[i] = (int(rng.integers(0, rows - nch + 1)), first, count, 0)
        if kind == "aligned":
            at = (at + 3) & ~3
        else:
            at += int(rng.integers(0, 2))  # odd and even columns
        cols[i] = at
        at += count
    stride = at | 1 if kind == "odd" else (at + 3) & ~3
    return w, cols, stride


def place(descs, planar, windows, cols, rows, stride, frames=None):
    """(int32 rows, float32 scale, mask): each frame's window of its planar block (at descs' out_offset in `planar`)
    placed at its rows and columns."""
    out = np.zeros((rows, stride), np.int32)
    scale = np.ones((rows, stride), np.float32)
    live = np.zeros((rows, stride), bool)
    for i in range(descs.size) if frames is None else frames:
        o, nch, bs = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]), int(descs[i]["block_size"])
        r, f, n, c = int(windows[i]["row"]), int(windows[i]["first"]), int(windows[i]["count"]), int(cols[i])
        out[r:r + nch, c:c + n] = planar[o:o + nch * bs].reshape(nch, bs)[:, f:f + n]
        scale[r:r + nch, c:c + n] = np.float32(2.0 ** -(int(descs[i]["bits_per_sample"]) - 1))
        live[r:r + nch, c:c + n] = True
    return out, scale, live


def as_mode(rows_i32, scale, mode):
    return rows_i32 if mode == I32 else rows_i32.astype(np.float32) * scale


def windowed(c, data, descs, windows, cols, rows, stride, mode):
    d = descs.copy()
    d["out_offset"] = cols
    dev = c.upload(data, d, mode=mode, channels=rows, channel_stride=stride, windows=windows)
    dev.decode(0)
    out, res = dev.read()
    dev.close()
    assert out.shape == (rows, stride)
    return out, res


def check(got, exp, live, what):
    g, e = bits(got), bits(exp)
    assert np.array_equal(g[live], e[live]), (what, np.argwhere((g != e) & live)[:8].tolist())
    assert not g[~live].any(), (what, "outside every window", np.argwhere((g != 0) & ~live)[:8].tolist())


def planar_of(b, descs):
    """The generator's PCM at descs' out_offset."""
    planar = np.zeros(int(descs["out_offset"][-1]) + int(descs["n_channels"][-1]) * int(descs["block_size"][-1]) + 4, np.int32)
    for i in range(b.n_frames):
        o, n = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]) * int(descs[i]["block_size"])
        planar[o:o + n] = b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])]
    return planar


def full_windows(descs):
    w = np.zeros(descs.size, dtype=cb.WINDOW_DTYPE)
    w["count"] = descs["block_size"]
    return w


# --------------------------------------------------------------------------- 1. full windows = channels batches

@gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_full_windows_equal_channels_batch(ctx, case):
    b = stream(case)
    descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    rows = int(descs["n_channels"].max())
    cols, stride = columns(descs, "packed")
    for mode in modes_for(descs):
        exp, eres = channels_batch(ctx, b.data, descs, cols, rows, stride, mode)
        got, res = windowed(ctx, b.data, descs, full_windows(descs), cols, rows, stride, mode)
        assert np.array_equal(res, eres), NAMES[mode]
        assert np.array_equal(bits(got), bits(exp)), NAMES[mode]


# --------------------------------------------------------------------------- 2. random windows against the oracle

@gpu
@pytest.mark.parametrize("kind", ["odd", "aligned"])
@pytest.mark.parametrize("case", sorted(CASES) + ["mixed"])
def test_random_windows_match_oracle(ctx, case, kind):
    if case == "mixed":
        b = F.mix(PARTS, seed=2024)
        descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
        ref = planar_of(b, descs)
    else:
        b = stream(case)
        descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
        st, ref = oracle_of(case, b.data, descs, b.frame_lengths, out_elems)
        assert (st == 0).all()
    rows = int(descs["n_channels"].max()) + 3
    w, cols, stride = random_windows(descs, rows, kind, seed=len(case))
    exp, scale, live = place(descs, ref, w, cols, rows, stride)
    for mode in modes_for(descs):
        out, res = windowed(ctx, b.data, descs, w, cols, rows, stride, mode)
        assert (res["status"] == 0).all() and np.array_equal(res["consumed"], b.frame_lengths), NAMES[mode]
        check(out, as_mode(exp, scale, mode), live, NAMES[mode])


# --------------------------------------------------------------------------- 3. neighbouring rows

@gpu
@pytest.mark.parametrize("name", ["c2", "c4-files", "mixed"])
def test_neighbouring_rows(ctx, name):
    """row_stride == count: rows packed back to back, so a store past a window's end would land in the next row's
    column 0.  The windows take the start, the end or the middle of each block; every byte is compared."""
    b = {"c2": lambda: synth.workload("c2", 96), "c4-files": lambda: stream("c4-files"),
         "mixed": lambda: F.mix(PARTS, seed=2024)}[name]()
    descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    planar = planar_of(b, descs)
    n = int(descs["block_size"].min()) - 1 | 1  # odd, shorter than every block
    w = np.zeros(descs.size, dtype=cb.WINDOW_DTYPE)
    nch = descs["n_channels"].astype(np.int64)
    w["row"] = np.concatenate([[0], np.cumsum(nch)[:-1]])
    bs = descs["block_size"].astype(np.int64)
    w["first"] = np.where(np.arange(descs.size) % 3 == 0, 0, np.where(np.arange(descs.size) % 3 == 1, bs - n, (bs - n) // 2))
    w["count"] = n
    rows = int(nch.sum())
    cols = np.zeros(descs.size, np.uint64)
    exp, scale, live = place(descs, planar, w, cols, rows, n)
    assert live.all()
    for mode in modes_for(descs):
        out, res = windowed(ctx, b.data, descs, w, cols, rows, n, mode)
        assert (res["status"] == 0).all(), NAMES[mode]
        assert np.array_equal(bits(out), bits(as_mode(exp, scale, mode))), NAMES[mode]


# --------------------------------------------------------------------------- 4. the fused writes alone, declined frames

@gpu
@pytest.mark.parametrize("no_wide", [False, True])
@pytest.mark.parametrize("case", ["c2-ms", "c4-files", "all-types-wasted-rice2", "8ch-12bit-fixed", "mixed"])
def test_fused_windows_alone(case, no_wide):
    c = cb.Context(device=0, lane_per_frame=True, no_generic=True, no_wide=no_wide)
    b = F.mix(PARTS, seed=2024) if case == "mixed" else stream(case)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    st, ref = oracle_of("alone-" + case, b.data, descs, b.frame_lengths, out_elems)
    _, pres = resident(c, b.data, descs, out_elems, cb.OUT_PLANAR_I32)
    rows = int(descs["n_channels"].max()) + 1
    w, cols, stride = random_windows(descs, rows, "aligned", seed=5)
    for mode in modes_for(descs):
        out, res = windowed(c, b.data, descs, w, cols, rows, stride, mode)
        assert np.array_equal(res["status"], pres["status"]), NAMES[mode]
        good = np.nonzero(res["status"] == 0)[0]
        assert good.size > 0
        exp, scale, live = place(descs, ref, w, cols, rows, stride, frames=good)
        g, e = bits(out), bits(as_mode(exp, scale, mode))
        assert np.array_equal(g[live], e[live]), NAMES[mode]
        _, _, any_live = place(descs, ref, w, cols, rows, stride)
        assert not g[~any_live].any(), NAMES[mode]
    c.close()


@gpu
@pytest.mark.parametrize("name", ["wrapping-mid-side", "corrupted"])
def test_declined_frames_inside_windows(ctx, name):
    """Frames the fast path declines (mid/side beyond 2^29, the corruption corpus): channels_kernel converts the
    planar batch's samples, inside each window only."""
    if name == "corrupted":
        data, offsets, lengths = corruption_corpus()
        descs, out_elems = cb.descs_from_offsets(data, offsets, lengths)
    else:
        b = synth.generate(WRAPPING_16)
        data = b.data
        descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    pout, pres = resident(ctx, data, descs, out_elems, cb.OUT_PLANAR_I32)
    rows = int(descs["n_channels"].max()) + 2
    w, cols, stride = random_windows(descs, rows, "odd", seed=9)
    exp, scale, live = place(descs, pout, w, cols, rows, stride)
    for mode in (I32, F32):
        out, res = windowed(ctx, data, descs, w, cols, rows, stride, mode)
        assert np.array_equal(res, pres), NAMES[mode]
        check(out, as_mode(exp, scale, mode), live, NAMES[mode])


# --------------------------------------------------------------------------- 5. adopted batches

@gpu
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_adopted_windowed_batch(config):
    import torch
    c = cb.Context(device=0, **CONFIGS[config])
    b = synth.workload("c2", 200)
    data = b.data.copy()
    victim = 77
    data[int(b.frame_offsets[victim]) + int(b.frame_lengths[victim]) - 3] ^= 0x01  # last data byte before the CRC-16
    descs, _ = cb.descs_from_offsets(data, b.frame_offsets[:-1], b.frame_lengths)
    t = torch.from_numpy(data).cuda()
    cols, stride = columns(descs, "packed")
    d = descs.copy()
    d["out_offset"] = cols
    w, wcols, wstride = random_windows(descs, 4, "odd", seed=3)
    dw = descs.copy()
    dw["out_offset"] = wcols
    planar = planar_of(b, descs)
    for mode in (I32, F32):
        dev = c.adopt(t.data_ptr(), t.numel(), d, mode=mode, channels=2, channel_stride=stride)
        n0 = c.launch_count
        dev.decode(0)
        n_ch = c.launch_count - n0
        dev.close()
        dev = c.adopt(t.data_ptr(), t.numel(), dw, mode=mode, channels=4, channel_stride=wstride, windows=w)
        n0 = c.launch_count
        dev.decode(0)
        assert c.launch_count - n0 == n_ch, NAMES[mode]
        out, res = dev.read()
        dev.close()
        if config == "lane-no-generic":
            continue
        assert res["status"][victim] == 23  # "frame CRC mismatch"
        good = [i for i in range(b.n_frames) if i != victim]
        assert (res["status"][good] == 0).all()
        exp, scale, live = place(descs, planar, w, wcols, 4, wstride, frames=good)
        g, e = bits(out), bits(as_mode(exp, scale, mode))
        assert np.array_equal(g[live], e[live]), NAMES[mode]
    c.close()


# --------------------------------------------------------------------------- 6. refusals

def create_windows(c, data, descs, windows, rows, stride, mode, n=None):
    h = C.c_void_p()
    st = c._L.clx_batch_create_windows(c._h, data.ctypes.data, data.size, descs.ctypes.data,
                                       None if windows is None else windows.ctypes.data,
                                       descs.size if n is None else n, rows, stride, 0, mode, C.byref(h))
    if st == 0:
        c._L.clx_batch_destroy(c._h, h)
    return st


@gpu
def test_refusals(ctx):
    b = synth.workload("c2", 8)
    descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    cols, stride = columns(descs, "packed")
    d = descs.copy()
    d["out_offset"] = cols
    w = full_windows(descs)
    bs = int(descs["block_size"][0])
    for mode in (I32, F32):
        assert create_windows(ctx, b.data, d, w, 2, stride, mode) == 0
        assert create_windows(ctx, b.data, d, w, 20, stride, mode) == 0  # no cap of 8 rows
        assert create_windows(ctx, b.data, d, None, 2, stride, mode) == 90
        assert create_windows(ctx, b.data, d[:0], None, 2, stride, mode, n=0) == 0  # no frames, no windows
        assert create_windows(ctx, b.data, d, w, 0, stride, mode) == 90
        assert create_windows(ctx, b.data, d, w, 2, 0, mode) == 90
        assert create_windows(ctx, b.data, d, w, 8, (1 << 64) // 16, mode) == 90  # 8 * stride * 4 overflows
        for field, value, rows in (("row", 1, 2), ("row", 3, 4), ("first", bs, 2), ("count", 0, 2),
                                   ("count", bs + 1, 2), ("reserved", 1, 2)):
            bad = w.copy()
            bad[field][3] = value
            if field == "row" and value == 1:
                assert create_windows(ctx, b.data, d, bad, rows, stride, mode) == 90  # row + 2 channels > 2 rows
                assert create_windows(ctx, b.data, d, bad, 3, stride, mode) == 0
            else:
                assert create_windows(ctx, b.data, d, bad, rows, stride, mode) == 90, (field, value)
        bad = w.copy()
        bad["first"][3], bad["count"][3] = 10, bs - 9  # first + count > block_size
        assert create_windows(ctx, b.data, d, bad, 2, stride, mode) == 90
        bad["count"][3] = bs - 10
        assert create_windows(ctx, b.data, d, bad, 2, stride, mode) == 0
        dd = d.copy()
        dd["out_offset"][-1] = stride - bs + 1  # column + count past the stride
        assert create_windows(ctx, b.data, dd, w, 2, stride, mode) == 90
        short = w.copy()
        short["count"][-1] = bs - 1  # the same column with one sample fewer fits
        assert create_windows(ctx, b.data, dd, short, 2, stride, mode) == 0
        far = d.copy()
        far["out_offset"][3] = (1 << 64) - 2  # column + count wraps
        assert create_windows(ctx, b.data, far, w, 2, stride, mode) == 90
        bad = d.copy()
        bad["byte_len"][2] = b.data.size  # beyond the bytes
        assert create_windows(ctx, b.data, bad, w, 2, stride, mode) == 90
        bad = d.copy()
        bad["n_channels"][1] = 0
        assert create_windows(ctx, b.data, bad, w, 2, stride, mode) == 90
    for mode in (cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I32, cb.OUT_INTERLEAVED_I16, cb.OUT_INTERLEAVED_I24, 6):
        assert create_windows(ctx, b.data, d, w, 2, stride, mode) == 90
    d25 = d.copy()
    d25["bits_per_sample"] = 25
    assert create_windows(ctx, b.data, d25, w, 2, stride, F32) == 90
    assert create_windows(ctx, b.data, d25, w, 2, stride, I32) == 0
    with pytest.raises(ValueError):
        ctx.upload(b.data, d, 2 * stride, windows=w)  # windows without a channel mode
    with pytest.raises(ValueError):
        ctx.upload(b.data, d, mode=I32, channels=2, channel_stride=stride, windows=w[:-1])


# --------------------------------------------------------------------------- 7. load_crops against slicing load()

def flac_file(name, n_frames):
    b = synth.workload(name, n_frames)
    return np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy()


def crop_of(full, o, n, C_):
    """load()'s [C_i, N] int32 / float32 rows cut to [C_, n] from column o, zeros past the end."""
    out = np.zeros((C_, n), full.dtype)
    part = full[:, o:o + n]
    out[:part.shape[0], :part.shape[1]] = part
    return out


@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_load_crops_match_slices(golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    srcs = [flac_file("c2", 40), flac_file("c4", 24)] + [golden[f"{n}__bytes"] for n in GOLDEN_AUDIO]
    idx = cb.index(srcs)
    fulls = [cb.load(s, dtype=dtype)[0].cpu().numpy() for s in srcs]
    assert [f.shape[1] for f in fulls] == [f.length for f in idx.files]
    rng = np.random.default_rng(17)
    bs0 = int(idx[0].descs["block_size"][0])
    files, offsets = [], []
    for fi, f in enumerate(idx.files):
        N = f.length
        starts = f.starts.tolist()
        cand = [0, N, N - 1, max(0, N - 3)]  # the whole file, the end, past the end
        if len(starts) > 2:
            cand += [starts[1], starts[2] - 1, starts[-1], starts[1] + 5]  # at and inside boundaries
        cand += rng.integers(0, N + 1, 4).tolist()
        for o in cand:
            if 0 <= o <= N:
                files.append(fi)
                offsets.append(int(o))
    for n in (1, 7, bs0 // 2, bs0, 3 * bs0 + 5, int(max(f.length for f in idx.files))):
        t, lengths = cb.load_crops(idx, files, offsets, n, dtype=dtype)
        C_ = max(f.info.channels for f in idx.files)
        assert t.shape == (len(files), C_, n) and t.dtype == dtype and t.is_cuda
        got = t.cpu().numpy()
        for b_, (fi, o) in enumerate(zip(files, offsets)):
            assert int(lengths[b_]) == min(n, idx[fi].length - o)
            assert np.array_equal(bits(got[b_]), bits(crop_of(fulls[fi], o, n, C_))), (fi, o, n)
    # overlapping excerpts of one file, B = 256 full-size excerpts
    t, _ = cb.load_crops(idx, [0] * 3, [100, 101, 4000], 5000, dtype=dtype)
    got = t.cpu().numpy()
    for b_, o in enumerate([100, 101, 4000]):
        assert np.array_equal(bits(got[b_]), bits(crop_of(fulls[0], o, 5000, 2)))


@gpu
def test_load_crops_full_size_batch():
    import torch
    srcs = [flac_file("c2", 300), flac_file("c2", 250)]
    idx = cb.index(srcs)
    fulls = [cb.load(s, dtype=torch.int32)[0].cpu().numpy() for s in srcs]
    rng = np.random.default_rng(4)
    n = 176400
    files = rng.integers(0, 2, 256)
    offsets = [int(rng.integers(0, idx[f].length - n)) for f in files]
    t, lengths = cb.load_crops(idx, files, offsets, n, dtype=torch.int32)
    assert t.shape == (256, 2, n) and (lengths == n).all()
    got = t.cpu().numpy()
    for b_, (fi, o) in enumerate(zip(files, offsets)):
        assert np.array_equal(got[b_], fulls[fi][:, o:o + n]), b_


@gpu
def test_load_crops_from_paths(golden, tmp_path):
    import torch
    paths = []
    for name in ("pop", "short"):
        p = tmp_path / f"{name}.flac"
        p.write_bytes(golden[f"{name}__bytes"].tobytes())
        paths.append(str(p))
    idx = cb.index(paths)
    assert isinstance(idx[0].data, np.memmap)
    t, lengths = cb.load_crops(idx, [0, 1], [10, 0], 300, dtype=torch.int32)
    for b_, p in enumerate(paths):
        full = cb.load(p, dtype=torch.int32)[0].cpu().numpy()
        o = [10, 0][b_]
        assert np.array_equal(t[b_].cpu().numpy(), crop_of(full, o, 300, 1))


# --------------------------------------------------------------------------- 8. load(frame_offset, num_frames)

@gpu
def test_load_frame_offset_matches_slices(golden):
    import torch
    srcs = [flac_file("c2", 30), flac_file("c4", 20)] + [golden[f"{n}__bytes"] for n in GOLDEN_AUDIO]
    for dtype in (torch.int32, torch.float32):
        fulls = [cb.load(s, dtype=dtype)[0] for s in srcs]
        for s, full in zip(srcs, fulls):
            N = full.shape[1]
            for o, n in ((0, -1), (0, 1), (min(5, N), 4096), (N // 2, -1), (N // 3, N), (N, -1), (N, 3)):
                t, _ = cb.load(s, dtype=dtype, frame_offset=o, num_frames=n)
                exp = full[:, o:] if n < 0 else full[:, o:o + n]
                assert t.shape == exp.shape and torch.equal(t, exp), (o, n)
        shortest = min(full.shape[1] for full in fulls)  # (a fixture holds 4 samples: a larger offset is refused)
        for o, n in ((0, -1), (min(3, shortest), 1000), (shortest, -1)):
            many = cb.load(srcs, dtype=dtype, frame_offset=o, num_frames=n)
            for (t, _), full in zip(many, fulls):
                exp = full[:, o:] if n < 0 else full[:, o:o + n]
                assert torch.equal(t, exp), (o, n)
    with pytest.raises(ValueError):
        cb.load(srcs[0], frame_offset=-1)
    with pytest.raises(ValueError):
        cb.load(srcs[0], frame_offset=fulls[0].shape[1] + 1)


@gpu
def test_consecutive_excerpts_give_the_streaminfo_md5(golden):
    import torch
    for name in ("pop", "short", "wasted_bits"):
        data = golden[f"{name}__bytes"]
        si, _ = cb.open_stream(data)
        N = cb.index(data)[0].length
        for step in (1000, 4097):
            parts = [cb.load(data, dtype=torch.int32, frame_offset=o, num_frames=step)[0].cpu().numpy()
                     for o in range(0, N, step)]
            pcm = np.concatenate(parts, axis=1)
            assert hashlib.md5(pcm.T.astype("<i2").tobytes()).digest() == si.md5sum, (name, step)
        idx = cb.index(data)
        offsets = list(range(0, N, 2000))
        t, lengths = cb.load_crops(idx, [0] * len(offsets), offsets, 2000, dtype=torch.int32)
        pcm = np.concatenate([t[b_, :si.channels, :int(lengths[b_])].cpu().numpy() for b_ in range(len(offsets))], axis=1)
        assert hashlib.md5(pcm.T.astype("<i2").tobytes()).digest() == si.md5sum, name


# --------------------------------------------------------------------------- 9. errors

@gpu
def test_crop_errors(golden):
    import torch
    data = flac_file("c4", 33)
    idx0 = cb.index(data)
    victim = 16
    d = idx0[0].descs[victim]
    data[int(d["byte_offset"]) + int(d["byte_len"]) // 2] ^= 0x10  # one corrupted frame in the middle
    with pytest.raises(cb.Error) as e_reader:
        list(cb.FlacReader.new(data).samples())
    idx = cb.index([golden["short__bytes"], data])
    f = idx[1]
    s0, bs = int(f.starts[victim]), int(f.descs["block_size"][victim])
    for dtype in (torch.int32, torch.float32):
        with pytest.raises(cb.Error) as e:
            cb.load_crops(idx, [0, 1, 1], [0, 0, s0 + bs - 10], 50, dtype=dtype)
        assert e.value == e_reader.value and "file 1, crop 2" in str(e.value)
        # the same corruption outside every excerpt: nothing to report
        t, _ = cb.load_crops(idx, [1, 1], [0, s0 + bs], 3 * bs, dtype=dtype)
        t, _ = cb.load_crops(idx, [1], [s0 - 10], 10, dtype=dtype)
        with pytest.raises(cb.Error) as e:
            cb.load(data, dtype=dtype, frame_offset=s0 - 10, num_frames=11)
        assert e.value == e_reader.value
        cb.load(data, dtype=dtype, frame_offset=s0 + bs)
    for args in (([0], [-1], 10), ([0], [idx[0].length + 1], 10), ([0], [0], 0), ([2], [0], 10), ([-1], [0], 10)):
        with pytest.raises(ValueError):
            cb.load_crops(idx, *args)
    with pytest.raises(ValueError):
        cb.load_crops(idx, [0], [0], 10, dtype=torch.int16)


# --------------------------------------------------------------------------- CPU: planner, index, exports

def descs_of(blocks, nch=2):
    d = np.zeros(len(blocks), dtype=cb.DESC_DTYPE)
    d["block_size"], d["n_channels"] = blocks, nch
    return d


def test_plan_range():
    d = descs_of([4096, 4096, 4096, 1001])
    assert cb.frame_starts(d).tolist() == [0, 4096, 8192, 12288]
    cases = {  # (lo, hi) -> [(frame, first, count)], column of lo = 7
        (0, 13289): [(0, 0, 4096), (1, 0, 4096), (2, 0, 4096), (3, 0, 1001)],
        (4096, 8192): [(1, 0, 4096)],
        (4095, 4097): [(0, 4095, 1), (1, 0, 1)],
        (100, 200): [(0, 100, 100)],
        (5000, 12300): [(1, 904, 3192), (2, 0, 4096), (3, 0, 12)],
        (13000, 20000): [(3, 712, 289)],
        (13289, 20000): [],
        (300, 300): [],
    }
    for (lo, hi), exp in cases.items():
        idx, w, cols = cb.plan_range(d, lo, hi, column=7, row=5)
        assert list(zip(idx.tolist(), w["first"].tolist(), w["count"].tolist())) == exp, (lo, hi)
        assert (w["row"] == 5).all() and (w["reserved"] == 0).all()
        starts = cb.frame_starts(d)[idx]
        assert (cols.astype(np.int64) == 7 + starts + w["first"].astype(np.int64) - lo).tolist() == [True] * idx.size
    idx, w, cols = cb.plan_range(descs_of([]), 0, 10)
    assert idx.size == 0 and w.size == 0 and cols.size == 0


def test_index_of_fixtures(golden):
    names = ["pop", "short", "wasted_bits"]
    idx = cb.index([golden[f"{n}__bytes"] for n in names])
    assert len(idx) == 3
    for f, n in zip(idx.files, names):
        pcm_len = golden[f"{n}__pcm"].size // f.info.channels
        assert f.length == pcm_len and f.end_confirmed
        assert f.starts.tolist() == cb.frame_starts(f.descs).tolist() and f.starts[0] == 0
        if f.info.samples:
            assert f.length == f.info.samples
    one = cb.index(golden["pop__bytes"])
    assert len(one) == 1 and one[0].length == idx[0].length
    with pytest.raises(cb.Error) as e:
        cb.index(golden["large_vendor_string__bytes"])
    assert e.value == cb.Error(43)
    odd = golden["pop__bytes"].copy()
    odd[20] ^= 0x02  # STREAMINFO channels 1 -> 2
    with pytest.raises(ValueError):
        cb.index([golden["short__bytes"], odd])


def test_window_entry_point_is_exported():
    """(CPU) clx_batch_create_windows is in the library's dynamic symbol table; WINDOW_DTYPE has the header's layout."""
    lib = C.CDLL(_lib.load()._name)
    assert hasattr(lib, "clx_batch_create_windows") and "clx_batch_create_windows" in _lib.SYMBOLS
    assert cb.WINDOW_DTYPE.itemsize == 16 == C.sizeof(_lib.FrameWindow)
    assert [cb.WINDOW_DTYPE.fields[n][1] for n in ("row", "first", "count", "reserved")] == [0, 4, 8, 12]
    for name in ("index", "load_crops", "WINDOW_DTYPE", "plan_range"):
        assert name in cb.__all__
