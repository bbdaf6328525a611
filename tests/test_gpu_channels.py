"""Channels-first i32 / f32 output of device-resident batches, and load() (-m gpu, except the CPU tests at the end).

A batch in CLX_OUT_CHANNELS_I32 / _F32 keeps one [rows, stride] buffer; out_offset is each frame's column.  On the
lane-per-frame path the decode kernel writes the rows itself and the frames the generic kernel takes over are
converted afterwards; every other path converts all frames inside the batch's graph.  Everything is compared with
the oracle's or the generator's PCM rearranged to rows on the host, and with the planar batch of the same frames.
"""
import ctypes as C
import hashlib

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from tests import fastpath as F
from tests.test_gpu_batch_out import CASES, WRAPPING_16, corruption_corpus, oracle_of, resident, stream
from tests.test_gpu_launch_sequence import CONFIGS
from tests.test_gpu_mixed import PARTS

gpu = pytest.mark.gpu

I32, F32 = cb.OUT_CHANNELS_I32, cb.OUT_CHANNELS_F32
NAMES = {I32: "i32", F32: "f32"}


def modes_for(descs):
    return [I32, F32] if int(descs["bits_per_sample"].max()) <= 24 else [I32]


def columns(descs, kind, seed=7):
    """(cols, stride) of a layout: frames packed from column 0, packed in a shuffled order, packed from column 3 with
    an odd stride, each on a multiple of 4 with the stride too, or 4-aligned with gaps of 8 columns between frames."""
    bs = descs["block_size"].astype(np.int64)
    order = np.arange(descs.size)
    if kind == "shuffled":
        order = np.random.default_rng(seed).permutation(descs.size)
    cols = np.zeros(descs.size, np.int64)
    at = 3 if kind == "odd" else 0
    for i in order:
        if kind in ("aligned", "gaps"):
            at = (at + 3) & ~3
        cols[i] = at
        at += int(bs[i]) + (8 if kind == "gaps" else 0)
    stride = at | 1 if kind == "odd" else (at + 3) & ~3 if kind in ("aligned", "gaps") else at
    return cols.astype(np.uint64), int(stride)


def to_rows(descs, planar, cols, rows, stride, frames=None):
    """(int32 [rows, stride], mask of covered elements): each frame's planar block (at descs' out_offset in `planar`)
    as rows at its column."""
    out = np.zeros((rows, stride), np.int32)
    live = np.zeros((rows, stride), bool)
    for i in range(descs.size) if frames is None else frames:
        o, nch, bs, c = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]), int(descs[i]["block_size"]), int(cols[i])
        out[:nch, c:c + bs] = planar[o:o + nch * bs].reshape(nch, bs)
        live[:nch, c:c + bs] = True
    return out, live


def scale_of(descs, cols, rows, stride):
    """float32 [rows, stride]: 2^-(bps-1) of the frame covering each element (1 where none does)."""
    s = np.ones((rows, stride), np.float32)
    for i in range(descs.size):
        bs, c = int(descs[i]["block_size"]), int(cols[i])
        s[:, c:c + bs] = np.float32(2.0 ** -(int(descs[i]["bits_per_sample"]) - 1))
    return s


def as_mode(rows_i32, scale, mode):
    return rows_i32 if mode == I32 else rows_i32.astype(np.float32) * scale


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def channels_batch(c, data, descs, cols, rows, stride, mode, stream_index=0):
    d = descs.copy()
    d["out_offset"] = cols
    dev = c.upload(data, d, mode=mode, channels=rows, channel_stride=stride)
    dev.decode(stream_index)
    out, res = dev.read()
    dev.close()
    assert out.shape == (rows, stride) and out.dtype == (np.float32 if mode == F32 else np.int32)
    return out, res


def check_equal(got, exp, live, what):
    g, e = bits(got), bits(exp)
    assert np.array_equal(g[live], e[live]), (what, np.argwhere((g != e) & live)[:8].tolist())


# --------------------------------------------------------------------------- 1. every path, every shape, both modes

@gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_channels_match_oracle_and_planar_batch(ctx, case):
    b = stream(case)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    st, ref = oracle_of(case, b.data, descs, b.frame_lengths, out_elems)
    assert (st == 0).all()
    pout, pres = resident(ctx, b.data, descs, out_elems, cb.OUT_PLANAR_I32)
    rows = int(descs["n_channels"].max())
    cols, stride = columns(descs, "packed")
    exp, live = to_rows(descs, ref, cols, rows, stride)
    fromplanar, _ = to_rows(descs, pout, cols, rows, stride)
    scale = scale_of(descs, cols, rows, stride)
    for mode in modes_for(descs):
        out, res = channels_batch(ctx, b.data, descs, cols, rows, stride, mode)
        assert np.array_equal(res, pres), NAMES[mode]
        assert (res["status"] == 0).all() and np.array_equal(res["consumed"], b.frame_lengths)
        check_equal(out, as_mode(exp, scale, mode), live, NAMES[mode])
        check_equal(out, as_mode(fromplanar, scale, mode), live, NAMES[mode])


# --------------------------------------------------------------------------- 2. column layouts

LAYOUT_STREAMS = {"c2": lambda: synth.workload("c2", 64), "c4-files": lambda: stream("c4-files"),
                  "mixed": lambda: F.mix(PARTS, seed=2024)}


@gpu
@pytest.mark.parametrize("kind", ["packed", "shuffled", "odd", "aligned", "gaps"])
@pytest.mark.parametrize("name", sorted(LAYOUT_STREAMS))
def test_column_layouts(ctx, name, kind):
    """Packed, shuffled and odd columns take the general flush; 4-aligned columns and stride let whole batches of one
    shape take the straight-line flush.  Elements between frames read 0."""
    b = LAYOUT_STREAMS[name]()
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    planar = np.zeros(out_elems, np.int32)
    for i in range(b.n_frames):
        o, n = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]) * int(descs[i]["block_size"])
        planar[o:o + n] = b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])]
    rows = int(descs["n_channels"].max())
    cols, stride = columns(descs, kind)
    exp, live = to_rows(descs, planar, cols, rows, stride)
    scale = scale_of(descs, cols, rows, stride)
    for mode in modes_for(descs):
        out, res = channels_batch(ctx, b.data, descs, cols, rows, stride, mode, stream_index=1)
        assert (res["status"] == 0).all(), NAMES[mode]
        check_equal(out, as_mode(exp, scale, mode), live, NAMES[mode])
        assert not bits(out)[~live].any(), NAMES[mode]  # gaps and rows a frame lacks: 0


# --------------------------------------------------------------------------- 3. mixed stream, 8 rows

@gpu
def test_mixed_stream_eight_rows(ctx):
    """1-8 channels, 8-24 bits, wasted bits, every stereo mode, shape_order reordering, in 8 rows: rows beyond a
    frame's channels read 0."""
    b = F.mix(PARTS, seed=2024)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    assert len(set(descs["n_channels"].tolist())) > 1 and len(set(descs["block_size"].tolist())) > 1
    planar = np.concatenate([b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])] for i in range(b.n_frames)])
    d2 = descs.copy()
    d2["out_offset"] = b.pcm_offsets[:-1]
    cols, stride = columns(descs, "packed")
    exp, live = to_rows(d2, planar, cols, 8, stride)
    scale = scale_of(descs, cols, 8, stride)
    for mode in (I32, F32):
        out, res = channels_batch(ctx, b.data, descs, cols, 8, stride, mode)
        assert (res["status"] == 0).all()
        check_equal(out, as_mode(exp, scale, mode), live, NAMES[mode])
        assert not bits(out)[~live].any()


# --------------------------------------------------------------------------- 4. the fused writes alone

@gpu
@pytest.mark.parametrize("no_wide", [False, True])
@pytest.mark.parametrize("case", ["c2-ms", "c2-indep", "c4-files", "all-types-wasted-rice2", "tiny-blocks-8bit",
                                  "8ch-12bit-fixed", "mixed"])
def test_fused_writes_alone(case, no_wide):
    c = cb.Context(device=0, lane_per_frame=True, no_generic=True, no_wide=no_wide)
    b = F.mix(PARTS, seed=2024) if case == "mixed" else stream(case)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    st, ref = oracle_of("alone-" + case, b.data, descs, b.frame_lengths, out_elems)
    _, pres = resident(c, b.data, descs, out_elems, cb.OUT_PLANAR_I32)
    rows = int(descs["n_channels"].max())
    cols, stride = columns(descs, "aligned")
    scale = scale_of(descs, cols, rows, stride)
    for mode in modes_for(descs):
        out, res = channels_batch(c, b.data, descs, cols, rows, stride, mode)
        assert np.array_equal(res["status"], pres["status"]), NAMES[mode]
        good = np.nonzero(res["status"] == 0)[0]
        assert good.size > 0
        exp, live = to_rows(descs, ref, cols, rows, stride, frames=good)
        check_equal(out, as_mode(exp, scale, mode), live, NAMES[mode])
    c.close()


# --------------------------------------------------------------------------- 5. frames the fused pass writes, then declines

@gpu
@pytest.mark.parametrize("name", ["wrapping-mid-side", "corrupted"])
def test_declined_frames_are_overwritten(ctx, name):
    if name == "corrupted":
        data, offsets, lengths = corruption_corpus()
        descs, out_elems = cb.descs_from_offsets(data, offsets, lengths)
    else:
        b = synth.generate(WRAPPING_16)
        data = b.data
        descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
        assert any(F.mid_side_beyond_bound(d, F.subframe_signals(data, d)) for d in descs)
    pout, pres = resident(ctx, data, descs, out_elems, cb.OUT_PLANAR_I32)
    if name == "corrupted":
        assert (pres["status"] != 0).sum() > 50
    rows = int(descs["n_channels"].max())
    cols, stride = columns(descs, "aligned")
    exp, live = to_rows(descs, pout, cols, rows, stride)
    scale = scale_of(descs, cols, rows, stride)
    for mode in (I32, F32):
        out, res = channels_batch(ctx, data, descs, cols, rows, stride, mode)
        assert np.array_equal(res, pres), NAMES[mode]
        check_equal(out, as_mode(exp, scale, mode), live, NAMES[mode])


# --------------------------------------------------------------------------- 6. the f32 rule, bit for bit

@gpu
@pytest.mark.parametrize("bps", [8, 12, 16, 20, 24])
def test_f32_bits(ctx, bps):
    cfg = synth.SynthConfig(n_frames=40, block_size=1152, n_channels=2, bps=bps, stereo_mode=-1, type_mask=15,
                            lpc_min_order=1, lpc_max_order=12, qlp_precision=0, rice_mode=-1, max_porder=3, wasted_max=2)
    b = synth.generate(cfg)
    descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    cols, stride = columns(descs, "aligned")
    i32, res = channels_batch(ctx, b.data, descs, cols, 2, stride, I32)
    f32, res2 = channels_batch(ctx, b.data, descs, cols, 2, stride, F32)
    assert (res["status"] == 0).all() and (res2["status"] == 0).all()
    assert np.array_equal(bits(f32), bits(i32.astype(np.float32) * np.float32(2.0 ** -(bps - 1))))
    # (the generator does not clamp to the nominal width: the samples of a valid stream are those within it)
    valid = (i32 >= -(1 << (bps - 1))) & (i32 < 1 << (bps - 1))
    assert valid.mean() > 0.5 and np.abs(i32[valid]).max() >= 1 << (bps - 3)  # the stream uses its width
    assert f32[valid].min() >= -1.0 and f32[valid].max() < 1.0


# --------------------------------------------------------------------------- 7. full size, many decodes

@gpu
@pytest.mark.parametrize("name,mode", [("c2", F32), ("c3", I32)])
def test_full_size_equals_generator(name, mode):
    c = cb.Context(device=0, lane_per_frame=True)
    b = synth.workload(name)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    rows = int(descs["n_channels"].max())
    cols, stride = columns(descs, "packed")
    exp, live = to_rows(descs, b.pcm, cols, rows, stride)
    assert live.all()
    exp = as_mode(exp, scale_of(descs, cols, rows, stride), mode)
    digest = hashlib.sha1(bits(exp).tobytes()).digest()
    d = descs.copy()
    d["out_offset"] = cols
    dev = c.upload(b.data, d, mode=mode, channels=rows, channel_stride=stride)
    for _ in range(2):
        dev.decode(0)
        out, res = dev.read()
        assert (res["status"] == 0).all() and np.array_equal(res["consumed"], b.frame_lengths)
        assert hashlib.sha1(bits(out).tobytes()).digest() == digest
        c.run_steps([dev], 50, 2)
        out, res = dev.read()
        assert (res["status"] == 0).all() and hashlib.sha1(bits(out).tobytes()).digest() == digest
    dev.close()
    c.close()


# --------------------------------------------------------------------------- 8. bytes in device memory, launch counts

@gpu
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_adopted_batch_crc_and_launches(config):
    import torch
    c = cb.Context(device=0, **CONFIGS[config])
    b = synth.workload("c2", 200)
    data = b.data.copy()
    victim = 77
    data[int(b.frame_offsets[victim]) + int(b.frame_lengths[victim]) - 3] ^= 0x01  # last data byte before the CRC-16
    descs, out_elems = cb.descs_from_offsets(data, b.frame_offsets[:-1], b.frame_lengths)
    t = torch.from_numpy(data).cuda()
    il = c.adopt(t.data_ptr(), t.numel(), descs, out_elems, mode=cb.OUT_INTERLEAVED_I32)
    n0 = c.launch_count
    il.decode(0)
    n_il = c.launch_count - n0
    il.close()
    cols, stride = columns(descs, "packed")
    d = descs.copy()
    d["out_offset"] = cols
    for mode in (I32, F32):
        dev = c.adopt(t.data_ptr(), t.numel(), d, mode=mode, channels=2, channel_stride=stride)
        n0 = c.launch_count
        dev.decode(0)
        assert c.launch_count - n0 == n_il, NAMES[mode]
        out, res = dev.read()
        dev.close()
        if config == "lane-no-generic":
            continue
        assert res["status"][victim] == 23  # "frame CRC mismatch"
        good = [i for i in range(b.n_frames) if i != victim]
        assert (res["status"][good] == 0).all()
        exp, live = to_rows(descs, b.pcm, cols, 2, stride, frames=good)
        check_equal(out, as_mode(exp, scale_of(descs, cols, 2, stride), mode), live, NAMES[mode])
    c.close()


# --------------------------------------------------------------------------- 9. refusals

def create_channels(c, data, descs, rows, stride, mode):
    h = C.c_void_p()
    st = c._L.clx_batch_create_channels(c._h, data.ctypes.data, data.size, descs.ctypes.data, descs.size, rows, stride,
                                        0, mode, C.byref(h))
    if st == 0:
        c._L.clx_batch_destroy(c._h, h)
    return st


@gpu
def test_refusals(ctx):
    b = synth.workload("c2", 8)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    cols, stride = columns(descs, "packed")
    d = descs.copy()
    d["out_offset"] = cols
    for mode in (I32, F32):
        assert create_channels(ctx, b.data, d, 2, stride, mode) == 0
        assert create_channels(ctx, b.data, d, 0, stride, mode) == 90
        assert create_channels(ctx, b.data, d, 9, stride, mode) == 90
        assert create_channels(ctx, b.data, d, 2, 0, mode) == 90
        assert create_channels(ctx, b.data, d, 8, (1 << 64) // 16, mode) == 90  # 8 * stride * 4 overflows
        assert create_channels(ctx, b.data, d, 1, stride, mode) == 90  # a frame has more channels than rows
        assert create_channels(ctx, b.data, d, 2, stride - 1, mode) == 90  # the last frame ends past the stride
        far = d.copy()
        far["out_offset"][3] = (1 << 64) - 2  # column + block_size wraps
        assert create_channels(ctx, b.data, far, 2, stride, mode) == 90
        bad = d.copy()
        bad["byte_len"][2] = b.data.size  # beyond the bytes
        assert create_channels(ctx, b.data, bad, 2, stride, mode) == 90
        bad = d.copy()
        bad["n_channels"][1] = 0
        assert create_channels(ctx, b.data, bad, 2, stride, mode) == 90
    for mode in (cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I32, cb.OUT_INTERLEAVED_I16, cb.OUT_INTERLEAVED_I24, 6):
        assert create_channels(ctx, b.data, d, 2, stride, mode) == 90
    d32 = d.copy()
    d32["bits_per_sample"] = 32  # a 32-bit frame (header value) in F32
    assert create_channels(ctx, b.data, d32, 2, stride, F32) == 90
    assert create_channels(ctx, b.data, d32, 2, stride, I32) == 0
    d25 = d.copy()
    d25["bits_per_sample"] = 25
    assert create_channels(ctx, b.data, d25, 2, stride, F32) == 90
    with pytest.raises(cb.Error) as e:
        ctx.upload(b.data, d, mode=F32, channels=1, channel_stride=stride)
    assert e.value.status == 90
    with pytest.raises(ValueError):
        ctx.upload(b.data, d, 2 * stride + 1, mode=F32, channels=2, channel_stride=stride)
    # the other calls keep refusing the channel modes
    for mode in (I32, F32):
        h = C.c_void_p()
        assert ctx._L.clx_batch_create_to(ctx._h, b.data.ctypes.data, b.data.size, descs.ctypes.data, descs.size,
                                          out_elems, 0, mode, C.byref(h)) == 90
        out = np.empty(out_elems, np.int32)
        results = np.zeros(descs.size, dtype=cb.RESULT_DTYPE)
        assert ctx._L.clx_decode_frames_to(ctx._h, b.data.ctypes.data, b.data.size, descs.ctypes.data, descs.size,
                                           out.ctypes.data, out_elems, results.ctypes.data, mode) == 90
    dev = ctx.upload(b.data, d, mode=I32, channels=2, channel_stride=stride)
    dev.decode(0)
    out = np.empty(2 * stride, np.int32)
    results = np.zeros(descs.size, dtype=cb.RESULT_DTYPE)
    assert ctx._L.clx_batch_read(ctx._h, dev._h, out.ctypes.data, out.size, results.ctypes.data) == 90
    part = np.zeros(2 * stride + 16, np.int32)
    assert ctx._L.clx_batch_read_to(ctx._h, dev._h, part.ctypes.data, part.size, results.ctypes.data) == 0
    full, _ = dev.read()
    assert np.array_equal(part[:2 * stride], full.reshape(-1)) and not part[2 * stride:].any()
    dev.close()


# --------------------------------------------------------------------------- 10. golden files through load()

GOLDEN_AUDIO = ["pop", "short", "wasted_bits", "empty_vorbis_comment", "repeated_vorbis_comment"]


def golden_rows(golden, name):
    """The committed PCM of a golden file as [channels, samples] int32, and its STREAMINFO."""
    data = golden[f"{name}__bytes"]
    si, first = cb.open_stream(data)
    descs, _, _, stop = cb.demux_frames(data, first)
    assert stop == cb.EOF
    pcm, at, blocks = golden[f"{name}__pcm"], 0, []
    for d in descs:
        nch, bs = int(d["n_channels"]), int(d["block_size"])
        blocks.append(pcm[at:at + nch * bs].reshape(nch, bs))
        at += nch * bs
    assert at == pcm.size
    return np.concatenate(blocks, axis=1).astype(np.int32), si


@gpu
def test_load_golden_files(golden):
    import torch
    exp = {name: golden_rows(golden, name) for name in GOLDEN_AUDIO}
    for name, (rows, si) in exp.items():
        data = golden[f"{name}__bytes"]
        t, sr = cb.load(data, dtype=torch.int32)
        assert t.is_cuda and t.dtype == torch.int32 and sr == si.sample_rate
        got = t.cpu().numpy()
        assert got.shape == rows.shape and np.array_equal(got, rows), name
        # interleaved back to little-endian i16: the file's own STREAMINFO MD5
        assert si.bits_per_sample == 16
        assert hashlib.md5(got.T.astype("<i2").tobytes()).digest() == si.md5sum, name
        f, sr = cb.load(bytes(data.tobytes()))  # float32 by default
        assert f.dtype == torch.float32 and sr == si.sample_rate
        fe = rows.astype(np.float32) * np.float32(2.0 ** -(si.bits_per_sample - 1))
        assert np.array_equal(bits(f.cpu().numpy()), bits(fe)), name
        assert f.numel() == 0 or (f.min().item() >= -1.0 and f.max().item() < 1.0), name
    srcs = [golden[f"{name}__bytes"] for name in GOLDEN_AUDIO]
    for dtype in (torch.int32, torch.float32):
        many = cb.load(srcs, dtype=dtype)
        assert len(many) == len(GOLDEN_AUDIO)
        for (t, sr), name in zip(many, GOLDEN_AUDIO):
            one, sr1 = cb.load(golden[f"{name}__bytes"], dtype=dtype)
            assert sr == sr1 and t.shape == one.shape and torch.equal(t, one), name
        base = many[0][0]
        assert all(t.untyped_storage().data_ptr() == base.untyped_storage().data_ptr() for t, _ in many)


@gpu
def test_load_path(golden, tmp_path):
    import torch
    p = tmp_path / "pop.flac"
    p.write_bytes(golden["pop__bytes"].tobytes())
    rows, si = golden_rows(golden, "pop")
    t, sr = cb.load(str(p), dtype=torch.int32)
    assert sr == si.sample_rate and np.array_equal(t.cpu().numpy(), rows)
    t2, _ = cb.load(p, dtype=torch.int32)
    assert torch.equal(t, t2)


# --------------------------------------------------------------------------- 11. load() errors

@gpu
def test_load_errors_match_flac_reader(golden):
    import torch
    b = synth.workload("c4", 33)
    data = np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy()  # 'fLaC' + STREAMINFO + 33 frames
    _, first = cb.open_stream(data)
    descs, _, _, _ = cb.demux_frames(data, first)
    assert descs.size == 33
    d = descs[descs.size // 2]
    data[int(d["byte_offset"]) + int(d["byte_len"]) // 2] ^= 0x10  # one corrupted frame in the middle
    with pytest.raises(cb.Error) as e_reader:
        list(cb.FlacReader.new(data).samples())
    for dtype in (torch.int32, torch.float32):
        with pytest.raises(cb.Error) as e_load:
            cb.load(data, dtype=dtype)
        assert e_load.value == e_reader.value
        with pytest.raises(cb.Error) as e_many:
            cb.load([golden["short__bytes"], data], dtype=dtype)
        assert e_many.value == e_reader.value and "file 1" in str(e_many.value)
    # the metadata error of the stream
    with pytest.raises(cb.Error) as e:
        cb.load(golden["large_vendor_string__bytes"])
    assert e.value == cb.Error(43)
    # a frame whose channel count differs from STREAMINFO's cannot be put in [C, N]
    odd = golden["pop__bytes"].copy()
    assert cb.open_stream(odd)[0].channels == 1
    odd[20] ^= 0x02  # STREAMINFO: channels - 1 (bits 3..1 of byte 20) from 0 to 1
    assert cb.open_stream(odd)[0].channels == 2
    with pytest.raises(ValueError):
        cb.load(odd)
    with pytest.raises(ValueError):
        cb.load(golden["pop__bytes"], dtype=torch.int16)


# --------------------------------------------------------------------------- 12. DeviceBatch.tensor()

@gpu
def test_tensor_waits_for_decode_stream():
    import torch
    c = cb.Context(device=0, lane_per_frame=True)
    b = synth.workload("c2", 512)
    descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    cols, stride = columns(descs, "packed")
    exp, _ = to_rows(descs, b.pcm, cols, 2, stride)
    d = descs.copy()
    d["out_offset"] = cols
    for mode in (I32, F32):
        dev = c.upload(b.data, d, mode=mode, channels=2, channel_stride=stride)
        dev.decode(1)  # internal stream 1; no sync before reading on torch's stream
        t = dev.tensor()
        assert t.shape == (2, stride) and t.is_cuda and t.data_ptr() == dev.device_out_ptr
        assert t.dtype == (torch.float32 if mode == F32 else torch.int32)
        got = t.clone().cpu().numpy()
        check_equal(got, as_mode(exp, scale_of(descs, cols, 2, stride), mode), np.ones(exp.shape, bool), NAMES[mode])
        del t
        dev.close()
    c.close()


# --------------------------------------------------------------------------- CPU: column planning, exports

def test_plan_columns():
    def descs_of(blocks, nch):
        d = np.zeros(len(blocks), dtype=cb.DESC_DTYPE)
        d["block_size"], d["n_channels"], d["out_offset"] = blocks, nch, 12345
        return d
    files = [descs_of([4096, 4096, 1001], 2), descs_of([16, 5], 6), descs_of([], 1), descs_of([4608], 1)]
    descs, starts, lengths, rows, stride = cb.plan_columns(files)
    assert lengths == [9193, 21, 0, 4608]
    assert starts == [0, 9196, 9220, 9220] and all(s % 4 == 0 for s in starts)
    assert stride == 13828 and stride % 4 == 0 and stride >= starts[-1] + lengths[-1]
    assert rows == 6
    assert descs["out_offset"].tolist() == [0, 4096, 8192, 9196, 9212, 9220]
    for s, n, d in zip(starts, lengths, files):  # every file's frames inside its own columns, back to back
        assert n == int(d["block_size"].sum())
    assert files[0]["out_offset"].tolist() == [12345] * 3  # the callers' arrays are left alone
    empty = cb.plan_columns([])
    assert empty[0].size == 0 and empty[1:] == ([], [], 0, 0)


def test_channel_modes_are_exported():
    """(CPU) clx_batch_create_channels is in the library's dynamic symbol table, and the mode values are the header's."""
    lib = C.CDLL(_lib.load()._name)
    assert hasattr(lib, "clx_batch_create_channels") and "clx_batch_create_channels" in _lib.SYMBOLS
    assert (cb.OUT_CHANNELS_I32, cb.OUT_CHANNELS_F32) == (4, 5)
    assert "load" in cb.__all__ and callable(cb.load)
