"""The catalogue of hand-written edge frames (tests/edge_frames.py) on the CPU.

Every entry is decoded by the Python restatement (tests/spec_decode.py) and by the oracle, and both must agree with
what the entry was built to decode to: status, PCM and bytes consumed.  That proves the writer and the expected
values before a GPU is involved.  Then the whole catalogue goes through the code the throughput path's kernels run
per lane (tools/seq_host.cpp over csrc/clx_lanes.h) at every head pad: it must accept every valid entry bit for bit
and never accept an invalid one.
"""
import ctypes as C

import numpy as np
import pytest

import claxon_b200 as cb
from oracle import oracle as O
from tests import edge_frames as E
from tests import fastpath as F
from tests import spec_decode
from tests.test_seq_host import harness, run_frames  # noqa: F401  (the lane harness fixture)

NAMES = [e.name for e in E.CATALOGUE]
SUBFRAME_ERRORS = range(11, 23)


def spec_status(msg: str) -> int:
    if msg == spec_decode.EOF_MSG:
        return E.EOF_ERR
    codes = {cb.status_str(c): c for c in range(3, 24)}
    return codes[msg]


@pytest.mark.parametrize("name", NAMES)
def test_entry_matches_spec_and_oracle(name):
    e = E.BY_NAME[name]
    kind, val = spec_decode.decode_frame(e.data)
    got = 0 if kind == "ok" else spec_status(val)
    assert got == e.status, (name, kind, val)
    o = O.decode_frame(e.data)
    assert o.status == e.status, (name, o.status)
    if e.status == E.OK:
        ch, consumed = val
        assert np.array_equal(np.array(ch, np.int64).reshape(-1), e.pcm.astype(np.int64)), name
        assert consumed == len(e.data)
        assert np.array_equal(o.samples, e.pcm) and o.info.consumed == len(e.data), name
    if e.status == E.CRC_MISMATCH:  # everything but the CRC-16 is right
        kind, val = spec_decode.decode_frame(e.data, verify_crc=False)
        assert kind == "ok" and np.array_equal(np.array(val[0], np.int64).reshape(-1), e.pcm.astype(np.int64))
        o = O.decode_frame(e.data, verify_crc=False)
        assert o.status == 0 and np.array_equal(o.samples, e.pcm)


def subframe_statuses(e: E.Entry) -> list[int]:
    """The oracle's status for each subframe of the frame in turn, up to the first that fails."""
    buf = np.frombuffer(e.data, np.uint8)
    pos = C.c_uint64(e.info["header_len"] * 8)
    bs = e.frame.bs
    out = []
    for ch in range(e.n_channels):
        x = np.empty(max(1, bs), np.int32)
        st = O.lib().clxo_decode_subframe(buf.ctypes.data, buf.size, C.byref(pos), E.sub_bits(e.frame, ch),
                                          x.ctypes.data_as(C.POINTER(C.c_int32)), bs)
        out.append(st)
        if st:
            break
    return out


@pytest.mark.parametrize("name", [e.name for e in E.CATALOGUE if e.channel is not None])
def test_error_sits_in_the_named_channel(name):
    e = E.BY_NAME[name]
    assert subframe_statuses(e) == [0] * e.channel + [e.status], name


def test_every_status_is_reached_where_named():
    reached = {e.status for e in E.CATALOGUE}
    assert {2, *range(11, 24)} <= reached, sorted({2, *range(11, 24)} - reached)
    for status in SUBFRAME_ERRORS:
        for nch in (3, 8):
            chans = {e.channel for e in E.CATALOGUE if e.status == status and e.n_channels == nch and "placed" in e.tags}
            assert chans == {0, nch // 2, nch - 1}, (status, nch, chans)


def test_catalogue_shapes():
    """What the entries were built to hold: the in-width tag says what keeps_width would, the pad-bit entries have
    0 and 7 pad bits, the accumulator entries sit on the i32 boundary, the full-scale ones reach both extremes."""
    for e in E.CATALOGUE:
        if e.status == 0:
            assert ("in-width" in e.tags) == e.in_width, e.name
    assert E.BY_NAME["shape/no-pad-bits"].info["pad"] == 0
    assert E.BY_NAME["shape/seven-pad-bits"].info["pad"] == 7
    classes = set()
    for e in E.CATALOGUE:
        if "acc-boundary" in e.tags:
            s = e.frame.subs[-1]
            b = E.sub_bits(e.frame, len(e.frame.subs) - 1)
            absum = sum(abs(c) for c in s.coefs)
            d = {"below": -1, "on": 0, "above": 1}[e.name.rsplit("/", 1)[1]]
            assert absum << (b - 1) == (1 << 31) + (d << (b - 1)), e.name
            classes.add(s.order)
        if "full-scale" in e.tags and not e.name.endswith("/constant"):  # (a constant holds one value)
            b = e.frame.bps
            assert e.pcm.min() <= -(1 << (b - 1)) and e.pcm.max() >= (1 << (b - 1)) - 1, e.name
    assert classes == {1, 8, 12, 32}


def test_warp_window_entries_are_predicted():
    """The three runs around the warp path's window limit: fastpath.warp_declines (exact for that path) declines
    exactly the runs that reach it, for a frame on a 16-byte boundary."""
    for d in (-1, 0, 1):
        e = E.BY_NAME[f"rice/warp-window{d:+d}"]
        data, offs, lens, _ = E.batch([e])
        descs, _ = cb.descs_from_offsets(data, offs, lens)
        assert F.warp_declines(data, descs[0]) == (d >= 0), d


def lane_verdicts(L, entries, head_pad, gaps=None):
    data, offs, lens, ref = E.batch(entries, gaps)
    descs, out, res = run_frames(L, data, offs, lens, head_pad)
    return descs, out, res, ref


@pytest.mark.parametrize("head_pad", range(16))
def test_lane_logic_on_catalogue(harness, head_pad):  # noqa: F811
    """Every valid entry is accepted bit-exact (status 0, consumed = length) and nothing invalid is accepted.  The
    lanes do not check the CRC-16 (a kernel of its own does), so a frame whose only fault is its CRC counts as valid
    here.  Frames sit at every byte offset mod 16 in turn."""
    entries = E.CATALOGUE
    gaps = [(i + head_pad) % 16 + 16 * (i == 0) for i in range(len(entries))]
    descs, out, res, ref = lane_verdicts(harness, entries, head_pad, gaps)
    for i, e in enumerate(entries):
        s = int(res["status"][i])
        if e.status in (E.OK, E.CRC_MISMATCH):
            assert s == 0, (e.name, head_pad, s)
            assert int(res["consumed"][i]) == len(e.data), e.name
            o, n = int(descs[i]["out_offset"]), e.pcm.size
            assert np.array_equal(out[o:o + n], e.pcm), (e.name, head_pad)
        else:
            assert s != 0, f"{e.name}: the lane accepted a frame the reference rejects with {e.status}"
