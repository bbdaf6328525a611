"""The catalogue of hand-written edge frames (tests/edge_frames.py) on the device (-m gpu).

Every entry's status and PCM are known by construction (and checked against two independent decoders by
test_edge_frames.py); here the device must reproduce them on every path (`ctx`: lane per frame, warp per frame,
generic kernel), through host-buffer calls and resident batches (uploaded, and adopted from device memory so that
the CRC-16 is checked on the device), in every output mode, and wherever the entry sits: alone, at lane 0 or 31 of a
warp of C2 frames, as a whole warp of copies, and at every byte offset mod 16.  With the fallback kernels switched
off, the fast paths' own verdicts must follow the rule of tests/fastpath.py: in particular every in-width valid entry
(full scale, the i32 accumulator boundary) comes back 0 from the fast path itself.
"""
import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from tests import edge_frames as E
from tests import fastpath as F

pytestmark = pytest.mark.gpu

PATHS = {"seq": dict(lane_per_frame=True), "warp": dict(warp_per_frame=True)}
ALL = E.CATALOGUE
SMALL = [e for e in ALL if "large" not in e.tags]
OFFSET_SUBSET = [e for e in ALL if e.tags & {"long-unary", "rice", "flush", "acc-boundary", "multichannel"}]


def decode(c, entries, route="host", gaps=None, mode=cb.OUT_PLANAR_I32):
    data, offs, lens, ref = E.batch(entries, gaps)
    descs, out_elems = cb.descs_from_offsets(data, offs, lens)
    if route == "host":
        out, res = c.decode_frames(data, descs, out_elems=out_elems, mode=mode)
    else:
        if route == "adopt":
            import torch
            t = torch.from_numpy(data).cuda()
            dev = c.adopt(t.data_ptr(), t.numel(), descs, out_elems, mode=mode)
        else:
            dev = c.upload(data, descs, out_elems, mode=mode)
        dev.decode(0)
        out, res = dev.read()
        dev.close()
    return data, descs, lens, ref, out, res


def check(entries, descs, out, res, what):
    for i, e in enumerate(entries):
        s = int(res["status"][i])
        assert s == e.status, (what, e.name, s, e.status)
        if e.status == 0:
            o = int(descs[i]["out_offset"])
            assert np.array_equal(out[o:o + e.pcm.size], e.pcm), (what, e.name)
            assert int(res["consumed"][i]) == len(e.data), (what, e.name)


# --------------------------------------------------------------------------- 1. every path, every route

@pytest.mark.parametrize("route", ["host", "upload", "adopt"])
def test_catalogue_on_every_path(ctx, route):
    gaps = [i % 16 for i in range(len(ALL))]
    _, descs, _, _, out, res = decode(ctx, ALL, route, gaps)
    check(ALL, descs, out, res, route)


# --------------------------------------------------------------------------- 2. the fast paths alone

@pytest.mark.parametrize("no_wide", [True, False], ids=["no-wide", "wide"])
@pytest.mark.parametrize("path", sorted(PATHS))
def test_fast_paths_alone(path, no_wide):
    c = cb.Context(device=0, no_generic=True, no_wide=no_wide, **PATHS[path])
    st = np.array([e.status for e in ALL], np.int32)
    for route in ("host", "upload"):
        data, descs, lens, ref, out, res = decode(c, ALL, route)
        F.check_fast_path(path, data, descs, lens, res, out, st, ref, wide_ran=not no_wide)
        for i, e in enumerate(ALL):
            if e.tags & {"full-scale", "acc-boundary"}:
                assert int(res["status"][i]) == 0, (path, route, e.name, int(res["status"][i]))
            if path == "seq" and "ms-bound" in e.tags and e.status == 0:
                beyond = max(abs(E.i32(v << s.wasted)) for s in e.frame.subs for v in s.signal) >= F.MID_SIDE_BOUND
                assert (int(res["status"][i]) != 0) == beyond, (e.name, int(res["status"][i]))
    c.close()


# --------------------------------------------------------------------------- 3. placement

def test_each_entry_alone(ctx):
    for e in ALL:
        _, descs, _, _, out, res = decode(ctx, [e])
        check([e], descs, out, res, "alone")


_c2 = []


def c2_frames():
    """31 C2 frames (16-bit mid/side, 4096 samples) as catalogue entries."""
    if not _c2:
        b = synth.workload("c2", 31)
        for i in range(b.n_frames):
            pcm = b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])]
            f = E.Frame(16, [E.Sub("constant", [0])] * 2, block_size=pcm.size // 2)
            _c2.append(E.Entry(f"c2/{i}", bytes(b.data[int(b.frame_offsets[i]):int(b.frame_offsets[i + 1])]), 0, pcm,
                               frame=f))
    return _c2


@pytest.mark.parametrize("where", ["lane0", "lane31", "warp"])
def test_placement_in_a_warp(ctx, where):
    """Entry i at lane 0 or lane 31 of the i-th group of 32 frames (the other 31 are C2 frames), or a whole group of
    32 copies of it: a warp's uniform choices (accumulator, order class, flush form) see the entry's shape."""
    c2 = c2_frames()
    for k in range(0, len(SMALL), 16):
        chunk = SMALL[k:k + 16]
        entries = []
        for e in chunk:
            entries += [e] * 32 if where == "warp" else [e] + c2 if where == "lane0" else c2 + [e]
        _, descs, _, _, out, res = decode(ctx, entries, "upload")
        check(entries, descs, out, res, where)


def test_byte_offsets(ctx):
    """Long unary runs, ring crossings, pairs, partitions of every length, at every residue mod 16."""
    for r in range(16):
        gaps, at = [], 0
        for e in OFFSET_SUBSET:
            gaps.append((r - at) % 16)
            at += gaps[-1] + len(e.data)
        data, descs, _, _, out, res = decode(ctx, OFFSET_SUBSET, "host", gaps)
        assert all(int(o) % 16 == r for o in descs["byte_offset"]), r
        check(OFFSET_SUBSET, descs, out, res, f"offset {r}")


# --------------------------------------------------------------------------- 4. output modes

ESIZE = {cb.OUT_INTERLEAVED_I32: 4, cb.OUT_INTERLEAVED_I24: 3, cb.OUT_INTERLEAVED_I16: 2}
IL_LIMIT = {cb.OUT_INTERLEAVED_I32: 32, cb.OUT_INTERLEAVED_I24: 24, cb.OUT_INTERLEAVED_I16: 16}


@pytest.mark.parametrize("route", ["host", "upload"])
@pytest.mark.parametrize("mode", sorted(ESIZE), ids=lambda m: {cb.OUT_INTERLEAVED_I32: "i32", cb.OUT_INTERLEAVED_I24: "i24",
                                                            cb.OUT_INTERLEAVED_I16: "i16"}[m])
def test_interleaved_modes(ctx, mode, route):
    entries = [e for e in SMALL if e.frame.bps <= IL_LIMIT[mode]]
    es = ESIZE[mode]
    data, descs, lens, ref, out, res = decode(ctx, entries, route, mode=mode)
    got = out.view(np.uint8)
    for i, e in enumerate(entries):
        assert int(res["status"][i]) == e.status, (e.name, int(res["status"][i]))
        if e.status == 0:
            o, n = int(descs[i]["out_offset"]), e.pcm.size
            exp = np.frombuffer(synth.interleaved_le_bytes(e.pcm, e.n_channels, 8 * es), np.uint8)
            assert np.array_equal(got[o * es:(o + n) * es], exp), e.name


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def as_mode(rows, bps, mode):
    return rows if mode == cb.OUT_CHANNELS_I32 else rows.astype(np.float32) * np.float32(2.0 ** -(bps - 1))


@pytest.mark.parametrize("mode", [cb.OUT_CHANNELS_I32, cb.OUT_CHANNELS_F32], ids=["ch-i32", "ch-f32"])
def test_channel_modes(ctx, mode):
    entries = SMALL
    data, offs, lens, _ = E.batch(entries)
    descs, _ = cb.descs_from_offsets(data, offs, lens)
    cols = np.concatenate([[0], np.cumsum([e.frame.bs for e in entries])[:-1]]).astype(np.uint64)
    stride = int(sum(e.frame.bs for e in entries))
    d = descs.copy()
    d["out_offset"] = cols
    dev = ctx.upload(data, d, mode=mode, channels=8, channel_stride=stride)
    dev.decode(0)
    out, res = dev.read()
    dev.close()
    for i, e in enumerate(entries):
        assert int(res["status"][i]) == e.status, (e.name, int(res["status"][i]))
        if e.status == 0:
            c, bs = int(cols[i]), e.frame.bs
            exp = as_mode(e.pcm.reshape(e.n_channels, bs), e.frame.bps, mode)
            assert np.array_equal(bits(out[:e.n_channels, c:c + bs]), bits(exp)), e.name


@pytest.mark.parametrize("mode", [cb.OUT_CHANNELS_I32, cb.OUT_CHANNELS_F32], ids=["ch-i32", "ch-f32"])
def test_windows_clip_full_scale_entries(ctx, mode):
    """Windows that drop the first and the last samples of every full-scale entry (a different amount each)."""
    entries = [e for e in ALL if "full-scale" in e.tags]
    data, offs, lens, _ = E.batch(entries)
    descs, _ = cb.descs_from_offsets(data, offs, lens)
    win = np.zeros(len(entries), cb.WINDOW_DTYPE)
    cols, at = [], 0
    for i, e in enumerate(entries):
        bs = e.frame.bs
        first = 1 + i % 3
        count = bs - first - 1 - i % 5
        win[i] = (2 * (i % 2), first, count, 0)
        cols.append(at)
        at += count
    d = descs.copy()
    d["out_offset"] = np.array(cols, np.uint64)
    dev = ctx.upload(data, d, mode=mode, channels=4, channel_stride=at, windows=win)
    dev.decode(0)
    out, res = dev.read()
    dev.close()
    assert (res["status"] == 0).all()
    for i, e in enumerate(entries):
        row, first, count = int(win[i]["row"]), int(win[i]["first"]), int(win[i]["count"])
        exp = as_mode(e.pcm.reshape(e.n_channels, e.frame.bs)[:, first:first + count], e.frame.bps, mode)
        got = out[row:row + e.n_channels, cols[i]:cols[i] + count]
        assert np.array_equal(bits(got), bits(exp)), e.name
