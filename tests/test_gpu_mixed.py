"""Batches that mix stream shapes (-m gpu, except the first test).

A resident batch built from several files, or one host-buffer call over several streams, puts frames of different
channel counts, bit depths and block sizes side by side.  Some code only such a mixture reaches: the device order
of shape_order() and the way results return to the caller's order (clx_decode_frames_to per chunk, clx_batch_read),
frames with fewer channels than the batch's channel slots (idle lanes, a stereo row pair next to a mono frame's in
pair_ca), the warp-wide choices all_narrow / any_wasted / fast_flush / order class over lanes of different bit
depths, and launch_interleave over frames of different widths.  Everything is checked frame by frame against the
generator's PCM and the oracle.
"""
import dataclasses

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from oracle import oracle as O
from tests import fastpath as F

gpu = pytest.mark.gpu

S = synth
# Optimal Rice everywhere, so that every frame keeps its nominal width (tests/fastpath.py).
PARTS = [
    S.SynthConfig(seed=11, n_frames=30, block_size=16, n_channels=1, bps=8, type_mask=15, lpc_min_order=1,
                  lpc_max_order=8, qlp_precision=0, rice_mode=-1, max_porder=2, wasted_max=2),
    S.SynthConfig(seed=12, n_frames=60, block_size=4096, n_channels=2, bps=16, stereo_mode=S.RANDOM_STEREO,
                  type_mask=12, lpc_min_order=1, lpc_max_order=12, qlp_precision=0, rice_mode=-1, max_porder=4,
                  rice2=2),
    # 24-bit mid/side with large samples, fixed and LPC subframes in the same warps (i32 and i64 accumulator lanes)
    S.SynthConfig(seed=13, n_frames=40, block_size=4608, n_channels=2, bps=24, stereo_mode=S.MID_SIDE,
                  type_mask=12, lpc_min_order=9, lpc_max_order=12, fixed_min_order=1, qlp_precision=15, rice_mode=-1,
                  max_porder=3, residual_mean=60000.0),
    S.SynthConfig(seed=14, n_frames=30, block_size=1152, n_channels=3, bps=20, type_mask=12, lpc_min_order=13,
                  lpc_max_order=32, qlp_precision=0, rice_mode=-1, max_porder=3, wasted_max=3),
    S.SynthConfig(seed=15, n_frames=30, block_size=192, n_channels=6, bps=12, type_mask=15, lpc_min_order=1,
                  lpc_max_order=8, qlp_precision=0, rice_mode=-1, max_porder=2, rice2=1),
    S.SynthConfig(seed=16, n_frames=20, block_size=1152, n_channels=8, bps=16, type_mask=12, lpc_min_order=1,
                  lpc_max_order=16, qlp_precision=0, rice_mode=-1, max_porder=2),
    S.SynthConfig(seed=17, n_frames=40, block_size=999, n_channels=2, bps=20, stereo_mode=S.RANDOM_STEREO,
                  type_mask=15, lpc_min_order=1, lpc_max_order=32, qlp_precision=0, rice_mode=-1, max_porder=0,
                  rice2=2, wasted_max=4),
    S.SynthConfig(seed=18, n_frames=40, block_size=192, n_channels=2, bps=12, stereo_mode=S.RANDOM_STEREO,
                  type_mask=12, lpc_min_order=1, lpc_max_order=8, qlp_precision=0, rice_mode=-1, max_porder=2),
]
# residuals drawn at a scale the bit depth leaves room for (the generator's default scale is for 16 bits and up)
PARTS = [dataclasses.replace(p, rice_kmax={8: 2, 12: 5, 16: 8, 20: 12, 24: 14}[p.bps]) for p in PARTS]
NARROW_PARTS = [p for p in PARTS if p.bps <= 16]


@pytest.fixture(scope="module")
def mixed():
    return F.mix(PARTS, seed=2024)


def descs_of(b):
    return cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)


def assert_frames(b, descs, out, res, expect=None):
    """Statuses at the caller's index (0 unless `expect` says otherwise), PCM of every good frame = generator."""
    expect = {} if expect is None else expect
    for i in range(b.n_frames):
        assert int(res["status"][i]) == expect.get(i, 0), (i, int(res["status"][i]))
        if i in expect:
            continue
        assert int(res["consumed"][i]) == int(b.frame_lengths[i]), i
        o, n = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]) * int(descs[i]["block_size"])
        lo, hi = int(b.pcm_offsets[i]), int(b.pcm_offsets[i + 1])
        assert np.array_equal(out[o:o + n], b.pcm[lo:hi]), f"frame {i} differs from the generator's PCM"


def test_mixed_stream_is_valid_by_construction(mixed):
    """(CPU) The mixture itself: every shape the GPU tests rely on is present, and the oracle decodes it frame by
    frame to the generator's PCM, every frame in its nominal width."""
    b = mixed
    descs, out_elems = descs_of(b)
    assert b.n_frames > 256
    assert set(descs["n_channels"].tolist()) == {1, 2, 3, 6, 8}
    assert set(descs["bits_per_sample"].tolist()) == {8, 12, 16, 20, 24}
    assert {16, 192, 1152, 4096, 4608, 999} <= set(descs["block_size"].tolist())
    assert set(descs["channel_assignment"][descs["n_channels"] == 2].tolist()) == {1, 8, 9, 10}
    bad, st, ref = O.decode_batch(b.data, b.frame_offsets[:-1], b.frame_lengths, descs["out_offset"], out_elems,
                                  n_threads=8)
    assert bad == 0
    res = np.zeros(b.n_frames, dtype=cb.RESULT_DTYPE)
    res["consumed"] = b.frame_lengths
    assert_frames(b, descs, ref, res)
    assert all(F.keeps_width(F.subframe_signals(b.data, d)) for d in descs)
    # every stream shape really is spread over the batch (no sorted runs of one shape)
    shapes = descs["n_channels"].astype(np.int64) * 100000 + descs["block_size"]
    assert (shapes[1:] != shapes[:-1]).mean() > 0.5


@gpu
def test_mixed_batch_host_call_every_path(ctx, mixed):
    """More than 256 frames on the context's two streams: two chunks, each reordered by shape on its own."""
    b = mixed
    descs, out_elems = descs_of(b)
    out, res = ctx.decode_frames(b.data, descs, out_elems=out_elems)
    assert_frames(b, descs, out, res)


@gpu
@pytest.mark.parametrize("path", ["seq", "warp"])
def test_mixed_batch_fast_paths_alone(path, mixed):
    """No valid frame is declined in a warp that mixes bit depths, channel counts, orders and stereo modes."""
    b = mixed
    descs, out_elems = descs_of(b)
    c = cb.Context(device=0, no_generic=True, no_wide=True,
                   **(dict(lane_per_frame=True) if path == "seq" else dict(warp_per_frame=True)))
    bad, st, ref = O.decode_batch(b.data, b.frame_offsets[:-1], b.frame_lengths, descs["out_offset"], out_elems,
                                  n_threads=8)
    out, res = c.decode_frames(b.data, descs, out_elems=out_elems)
    v = F.check_fast_path(path, b.data, descs, b.frame_lengths, res, out, st, ref, wide_ran=False)
    assert v.declined == 0 and v.out_of_width == 0
    assert_frames(b, descs, out, res)
    dev = c.upload(b.data, descs, out_elems)
    dev.decode(0)
    out2, res2 = dev.read()
    dev.close()
    assert_frames(b, descs, out2, res2)
    c.close()


@gpu
@pytest.mark.parametrize("layout", ["packed-odd", "aligned-16-byte", "reversed"])
def test_mixed_batch_output_layouts(ctx, mixed, layout):
    """Caller-chosen out_offsets: packed back to back from an odd element, every frame on a 16-byte boundary, or
    in reverse frame order (not stream order: one chunk)."""
    b = mixed
    descs, _ = descs_of(b)
    sizes = descs["n_channels"].astype(np.uint64) * descs["block_size"].astype(np.uint64)
    if layout == "packed-odd":
        offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint64) + np.uint64(3)
    elif layout == "aligned-16-byte":
        padded = (sizes + np.uint64(3)) & ~np.uint64(3)
        offs = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.uint64) + np.uint64(4)
    else:
        rev = sizes[::-1]
        offs = np.concatenate([[0], np.cumsum(rev)[:-1]]).astype(np.uint64)[::-1] + np.uint64(1)
    descs["out_offset"] = offs
    total = int((offs + sizes).max())
    out = np.full(total + 2, 77, dtype=np.int32)
    out, res = ctx.decode_frames(b.data, descs, out=out, out_elems=total + 2)
    assert_frames(b, descs, out, res)
    covered = np.zeros(out.size, bool)
    for o, n in zip(offs.tolist(), sizes.tolist()):
        covered[o:o + n] = True
    if layout != "aligned-16-byte":  # (alignment gaps inside the call's range are unspecified)
        assert (out[~covered] == 77).all()
    else:
        assert out[0] == 77 and out[-1] == 77


@gpu
def test_mixed_resident_batch_two_streams_and_adopt(ctx, mixed):
    """The resident batch keeps a device order of its own (shape_order over the whole batch): decoded on two
    different streams one after the other, read back, every status and `consumed` at the caller's index.  The same
    from device bytes (adopt), whose CRC-16 runs on the device over the sorted descriptors."""
    import torch
    b = mixed
    descs, out_elems = descs_of(b)
    dev = ctx.upload(b.data, descs, out_elems)
    for s in (0, 1):
        dev.decode(s)
        dev.sync()
        out, res = dev.read()
        assert_frames(b, descs, out, res)
    dev.close()
    t = torch.from_numpy(b.data.copy()).cuda()
    dev = ctx.adopt(t.data_ptr(), t.numel(), descs, out_elems)
    dev.decode(1)
    out, res = dev.read()
    dev.close()
    assert_frames(b, descs, out, res)


def damaged(b, descs):
    """Flips the first subframe's pad bit of one frame of each of several shapes ("invalid subframe header", 11)
    and a residual bit of two more ("frame CRC mismatch", 23)."""
    data = b.data.copy()
    expect, seen = {}, set()
    for i in range(b.n_frames):
        shape = (int(descs[i]["n_channels"]), int(descs[i]["block_size"]), int(descs[i]["bits_per_sample"]))
        if shape in seen or i % 3:
            continue
        seen.add(shape)
        off = int(b.frame_offsets[i])
        if len(seen) % 4 == 0:
            data[off + int(b.frame_lengths[i]) - 3] ^= 0x01  # last data byte before the CRC-16
            expect[i] = 23
        else:
            data[off + int(descs[i]["header_len"])] ^= 0x80
            expect[i] = 11
    assert len(seen) >= 6
    return data, expect


@gpu
def test_mixed_batch_damaged_frames_keep_their_index(ctx, mixed):
    """Damaged frames of different shapes: their statuses come back at the caller's index, through the host-buffer
    call and through a resident batch, and their neighbours are intact."""
    b = mixed
    descs, out_elems = descs_of(b)
    data, expect = damaged(b, descs)
    bad, st, ref = O.decode_batch(data, b.frame_offsets[:-1], b.frame_lengths, descs["out_offset"], out_elems,
                                  n_threads=8)
    for i in range(b.n_frames):  # the damage means to the oracle what it is meant to
        assert int(st[i]) == expect.get(i, 0), (i, int(st[i]))
    dd = cb.descs_from_offsets(data, b.frame_offsets[:-1], b.frame_lengths)[0]
    out, res = ctx.decode_frames(data, dd, out_elems=out_elems)
    assert_frames(b, dd, out, res, expect)
    dev = ctx.upload(data, dd, out_elems)
    dev.decode(1)
    out, res = dev.read()
    dev.close()
    assert_frames(b, dd, out, res, expect)


def interleaved_expected(b, descs, out_elems):
    exp = np.zeros(out_elems, dtype=np.int64)
    for i in range(b.n_frames):
        o, nch, bs = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]), int(descs[i]["block_size"])
        lo, hi = int(b.pcm_offsets[i]), int(b.pcm_offsets[i + 1])
        exp[o:o + nch * bs] = b.pcm[lo:hi].reshape(nch, bs).T.reshape(-1)
    return exp


@gpu
def test_mixed_batch_interleaved_modes(ctx, mixed):
    """I32 and I24 for the mixture up to 24 bits, I16 for a mixture of 8 to 16 bits, frame widths side by side
    in one launch_interleave; one 20-bit frame makes a whole I16 call invalid."""
    b = mixed
    descs, out_elems = descs_of(b)
    exp = interleaved_expected(b, descs, out_elems)
    live = np.zeros(out_elems, dtype=bool)
    for d in descs:
        live[int(d["out_offset"]):int(d["out_offset"]) + int(d["n_channels"]) * int(d["block_size"])] = True
    out32, res = ctx.decode_frames(b.data, descs, out_elems=out_elems, mode=cb.OUT_INTERLEAVED_I32)
    assert (res["status"] == 0).all() and np.array_equal(out32[:out_elems][live], exp[live])
    out24, res = ctx.decode_frames(b.data, descs, out_elems=out_elems, mode=cb.OUT_INTERLEAVED_I24)
    got = out24[:3 * out_elems].reshape(-1, 3).astype(np.int64)
    val = got[:, 0] | (got[:, 1] << 8) | (got[:, 2] << 16)
    val = (val ^ 0x800000) - 0x800000
    assert (res["status"] == 0).all() and np.array_equal(val[live], exp[live])
    with pytest.raises(cb.Error) as e:
        ctx.decode_frames(b.data, descs, out_elems=out_elems, mode=cb.OUT_INTERLEAVED_I16)
    assert e.value.status == 90

    n = F.mix(NARROW_PARTS, seed=7)
    nd, n_elems = descs_of(n)
    assert set(nd["bits_per_sample"].tolist()) == {8, 12, 16}
    nexp = interleaved_expected(n, nd, n_elems)
    nlive = np.zeros(n_elems, dtype=bool)
    for d in nd:
        nlive[int(d["out_offset"]):int(d["out_offset"]) + int(d["n_channels"]) * int(d["block_size"])] = True
    out16, res = ctx.decode_frames(n.data, nd, out_elems=n_elems, mode=cb.OUT_INTERLEAVED_I16)
    assert out16.dtype == np.int16 and (res["status"] == 0).all()
    assert np.array_equal(out16[:n_elems][nlive].astype(np.int64), nexp[nlive])
    # one 20-bit frame among them: the whole call is refused
    wide = F.mix(NARROW_PARTS + [S.SynthConfig(seed=19, n_frames=1, block_size=192, n_channels=2, bps=20,
                                               type_mask=8, lpc_min_order=1, lpc_max_order=8, rice_mode=-1)], seed=7)
    wd, w_elems = descs_of(wide)
    with pytest.raises(cb.Error) as e:
        ctx.decode_frames(wide.data, wd, out_elems=w_elems, mode=cb.OUT_INTERLEAVED_I16)
    assert e.value.status == 90
