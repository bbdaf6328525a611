"""What the fast paths must decode by themselves, checked frame by frame (test helper, no tests here).

Under Context(no_generic=True, no_wide=True) nothing repairs a fast path's verdict: a frame the warp-per-frame path
(csrc/clx_coop.cu) or the lane-per-frame path (csrc/clx_fused.cu) declines comes back with -2 (the generic kernel
would have decoded it) or -3 (the lane-per-frame path's i64 second chance would have).  The rule those verdicts must
follow comes from the exactness bounds in the two files:

  * A frame "keeps its nominal width" when every subframe signal the decoder reconstructs — each channel, or
    left/side, side/right, mid/side, after the wasted-bits shift — lies in [-2^(b-1), 2^(b-1)), b being the frame's
    bit depth plus one for a side channel.  The i32 accumulator is exact for such a frame and the mid/side bound
    (2^29) is far away, so both fast paths must return status 0 for it, bit-exact, `consumed` = frame length.
  * A frame that leaves its nominal width may come back -2 or -3 (lane per frame) or -2 (warp per frame).  A
    mid/side frame with a subframe signal of magnitude >= 2^29 cannot be 0 on the lane-per-frame path, and once the
    i64 second chance has run (no_wide=False) it is exactly -2.
  * The warp-per-frame path decodes a partition's Rice codes one 128-word window at a time and needs every code's
    unary terminator inside the first 127 words of the window that starts at the code's 128-bit-aligned position
    (rice_window): a code whose unary run is 4064 - (start bit mod 128) bits or longer is declined (-2), whatever
    the frame's width.  `warp_declines` predicts exactly that.
  * A frame the oracle rejects never comes back with status 0.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from claxon_b200 import synth
from oracle import oracle as O

NEED_GENERIC, NEED_WIDE = -2, -3
WARP_WINDOW_BITS = 127 * 32   # bits of a 128-word window that may hold a code's terminator
MID_SIDE_BOUND = 1 << 29


def subframe_signals(data, desc) -> list[np.ndarray]:
    """The subframe signals of a frame the oracle accepts, decoded one subframe at a time by the oracle (i32, after
    the wasted-bits shift), with the bit depth each one is coded with."""
    buf = np.ascontiguousarray(data, dtype=np.uint8)
    off, n = int(desc["byte_offset"]), int(desc["byte_len"])
    bs, nch, ca, bps = int(desc["block_size"]), int(desc["n_channels"]), int(desc["channel_assignment"]), \
        int(desc["bits_per_sample"])
    pos = C.c_uint64(int(desc["header_len"]) * 8)
    sig = []
    for ch in range(nch):
        b = bps + (1 if (ca == 9 and ch == 0) or (ca in (8, 10) and ch == 1) else 0)
        x = np.empty(bs, np.int32)
        st = O.lib().clxo_decode_subframe(buf.ctypes.data + off, n, C.byref(pos), b,
                                          x.ctypes.data_as(C.POINTER(C.c_int32)), bs)
        assert st == 0, (st, ch)
        sig.append((x, b))
    return sig


def keeps_width(sig) -> bool:
    return all(int(x.min()) >= -(1 << (b - 1)) and int(x.max()) < (1 << (b - 1)) for x, b in sig)


def mid_side_beyond_bound(desc, sig) -> bool:
    return int(desc["channel_assignment"]) == 10 and max(int(np.abs(x.astype(np.int64)).max()) for x, _ in sig) \
        >= MID_SIDE_BOUND


# --------------------------------------------------------------------------- warp-per-frame window limit

def _walk(bits: np.ndarray, nxt: list, desc, base_bit: int) -> bool:
    """True if some Rice code of the (valid) frame has a unary run the warp-per-frame window cannot hold."""
    def rd(p, n):
        v = 0
        for x in bits[p:p + n].tolist():
            v = (v << 1) | x
        return v
    bs, nch, ca, bps = int(desc["block_size"]), int(desc["n_channels"]), int(desc["channel_assignment"]), \
        int(desc["bits_per_sample"])
    p = int(desc["header_len"]) * 8
    for ch in range(nch):
        b = bps + (1 if (ca == 9 and ch == 0) or (ca in (8, 10) and ch == 1) else 0)
        head = rd(p, 8)
        p += 8
        code = (head >> 1) & 63
        if head & 1:  # wasted bits, unary coded: warm-up / verbatim samples are that much narrower
            one = nxt[p]
            b -= one - p + 1
            p = one + 1
        if code == 0:
            p += b
            continue
        if code == 1:
            p += bs * b
            continue
        order = code & 7 if (code & 0x38) == 0x08 else (code & 31) + 1
        p += order * b
        if (code & 0x38) != 0x08:  # LPC: precision, shift, coefficients
            p += 9 + order * (rd(p, 4) + 1)
        method, po = rd(p, 2), rd(p + 2, 4)
        p += 6
        pbits, per = (4 if method == 0 else 5), bs >> po
        for part in range(1 << po):
            k = rd(p, pbits)
            p += pbits
            for _ in range(per - order if part == 0 else per):
                one = nxt[p]
                if one - p >= WARP_WINDOW_BITS - ((base_bit + p) & 127):
                    return True
                p = one + 1 + k
    return False


def warp_declines(data, desc) -> bool:
    """Exact prediction of rice_window's limit in clx_coop.cu for a frame the oracle accepts."""
    off, n = int(desc["byte_offset"]), int(desc["byte_len"])
    bits = np.unpackbits(np.ascontiguousarray(data[off:off + n], dtype=np.uint8))
    ones = np.flatnonzero(bits)
    # cheap filter: no zero run long enough, no code long enough
    gaps = np.diff(np.concatenate([[-1], ones, [bits.size]]))
    if gaps.max() - 1 < WARP_WINDOW_BITS - 127 - 31:
        return False
    idx = np.searchsorted(ones, np.arange(bits.size + 1))
    nxt = np.where(idx < ones.size, ones[np.minimum(idx, ones.size - 1)], bits.size + (1 << 20)).tolist()
    return _walk(bits, nxt, desc, (off & 15) * 8)


# --------------------------------------------------------------------------- the rule

@dataclass
class Verdicts:
    out_of_width: int = 0   # oracle-accepted frames that leave their nominal width
    declined: int = 0       # frames with status -2 / -3
    wide: int = 0           # frames with status -3
    warp_long: int = 0      # frames declined for the warp window limit


def check_fast_path(path: str, data, descs, lengths, res, out, st, ref, wide_ran: bool) -> Verdicts:
    """Asserts the rule of this module for every frame of one decode under no_generic (and no_wide unless
    `wide_ran`).  `path`: "seq" (lane per frame) or "warp" (warp per frame); st / ref: the oracle's statuses and
    planar PCM at descs' out_offsets; lengths: the bytes each accepted frame consumes."""
    v = Verdicts()
    status = res["status"]
    for i in range(len(descs)):
        d, s = descs[i], int(status[i])
        if s in (NEED_GENERIC, NEED_WIDE):
            v.declined += 1
            v.wide += s == NEED_WIDE
        assert s != NEED_WIDE or (path == "seq" and not wide_ran), (path, i, s)
        if st[i] != 0:
            assert s != 0, f"frame {i}: the {path} path accepted a frame the oracle rejects with {st[i]}"
            assert s < 0 or s == st[i], (i, s, st[i])  # a status of its own must be the oracle's
            continue
        sig = subframe_signals(data, d)
        keeps = keeps_width(sig)
        v.out_of_width += not keeps
        long = path == "warp" and warp_declines(data, d)
        v.warp_long += long
        if long:
            assert s == NEED_GENERIC, f"frame {i}: a Rice code longer than the window, expected -2, got {s}"
        elif keeps:
            assert s == 0, f"frame {i} ({path}) keeps its nominal width but came back {s}"
        elif path == "seq" and mid_side_beyond_bound(d, sig):
            assert s == NEED_GENERIC or (s == NEED_WIDE and not wide_ran), \
                f"frame {i}: mid/side beyond 2^29 came back {s}"
        else:
            assert s in (0, NEED_GENERIC, NEED_WIDE), (i, s)
        if s == 0:
            o, n = int(d["out_offset"]), int(d["n_channels"]) * int(d["block_size"])
            assert np.array_equal(out[o:o + n], ref[o:o + n]), f"frame {i} ({path}) differs from the oracle"
            assert int(res["consumed"][i]) == int(lengths[i]), (i, int(res["consumed"][i]), int(lengths[i]))
    return v


# --------------------------------------------------------------------------- batches that mix stream shapes

def mix(configs: list[synth.SynthConfig], seed: int) -> synth.SynthBatch:
    """One stream out of the frames of several SynthConfigs, in a seeded random order.  Frames are
    self-contained, so the result decodes frame by frame to the concatenated PCM in the new order."""
    parts = [synth.generate(c) for c in configs]
    frames = [(p, i) for p in parts for i in range(p.n_frames)]
    order = np.random.default_rng(seed).permutation(len(frames))
    data, pcm = [], []
    for j in order:
        p, i = frames[j]
        data.append(p.data[int(p.frame_offsets[i]):int(p.frame_offsets[i + 1])])
        pcm.append(p.pcm[int(p.pcm_offsets[i]):int(p.pcm_offsets[i + 1])])
    offs = np.concatenate([[0], np.cumsum([x.size for x in data])]).astype(np.uint64)
    poffs = np.concatenate([[0], np.cumsum([x.size for x in pcm])]).astype(np.uint64)
    return synth.SynthBatch(configs[0], np.concatenate(data), offs, np.concatenate(pcm), poffs,
                            meta={"configs": configs, "seed": seed})
