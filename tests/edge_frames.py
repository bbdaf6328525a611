"""FLAC frames written field by field at the format's limits, with the PCM they decode to known by construction
(test helper, no tests here).

The frames the rest of the suite decodes come from csrc/synth.c or from libFLAC, and neither goes near the places
where the kernels make exactness decisions: samples at -2^(b-1) or 2^(b-1) - 1, sum|coef| << (b-1) on 2^31, mid/side
subframes at 2^29, Rice codes exactly 32 bits long, unary runs across the rings, escape parameters, empty
partitions, every subframe-level error in a chosen channel.  This module writes such frames from the frame layout
as the reference decoder reads it (src/frame.rs, src/subframe.rs), sharing nothing with synth.c.

A subframe is described by its TARGET signal (the values before the wasted-bits shift) and its predictor; the writer
computes each residual so that the reference recurrence reproduces the target (i64 sum, arithmetic shift and a
wrapping i32 add for LPC, wrapping i32 for fixed), so any signal is encodable with any predictor.  The expected
output is the targets after the wasted-bits shift, with the stereo decorrelation undone as src/frame.rs:319-389 does.

Escape hatches for invalid frames: a raw override of every field (reserved values, escape parameters, a negative
shift, precision code 15, pad bits), truncation and a wrong CRC-16.  CRC-8 and CRC-16 are computed otherwise.

    CATALOGUE: list[Entry]       every entry, by name: frame bytes, expected status, expected planar PCM
    batch(frames, ...)           frames laid out in one byte buffer, with the expected PCM at descs' out_offsets
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace

import numpy as np

M32 = 0xFFFFFFFF
RICE_ESCAPE = {0: 15, 1: 31}
BPS_CODE = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6}
FIXED = {0: (), 1: (1,), 2: (2, -1), 3: (3, -3, 1), 4: (4, -6, 4, -1)}  # c[j] multiplies s[t-1-j]

OK, EOF_ERR = 0, 2
PAD_BIT, SUB_RESERVED, WASTED_GT_31, NO_NON_WASTED = 11, 12, 13, 14
RES_RESERVED, PORDER_INVALID, RES_INVALID, ESCAPE = 15, 16, 17, 18
FIXED_GT_BLOCK, LPC_GT_BLOCK, PRECISION_INVALID, NEGATIVE_SHIFT, CRC_MISMATCH = 19, 20, 21, 22, 23


def i32(v: int) -> int:
    v &= M32
    return v - (1 << 32) if v & 0x80000000 else v


def crc8(data: bytes) -> int:
    crc = 0
    for byte in data:
        crc ^= byte
        for _ in range(8):
            crc = ((crc << 1) ^ 0x07) & 0xFF if crc & 0x80 else (crc << 1) & 0xFF
    return crc


def crc16(data: bytes) -> int:
    crc = 0
    for byte in data:
        crc ^= byte << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x8005) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return crc


class BitWriter:
    """MSB-first."""

    def __init__(self):
        self.bits: list[int] = []

    def put(self, v: int, n: int):
        assert n == 0 or 0 <= v < (1 << n), (v, n)
        self.bits.extend((v >> (n - 1 - i)) & 1 for i in range(n))

    def put_signed(self, v: int, n: int):
        assert -(1 << (n - 1)) <= v < (1 << (n - 1)), (v, n)
        self.put(v & ((1 << n) - 1), n)

    def unary(self, q: int):
        self.bits.extend([0] * q)
        self.bits.append(1)

    def __len__(self):
        return len(self.bits)

    def to_bytes(self, fill: int = 0) -> tuple[bytes, int]:
        pad = -len(self.bits) % 8
        bits = self.bits + [fill] * pad
        return np.packbits(np.array(bits, np.uint8)).tobytes(), pad


# --------------------------------------------------------------------------- description of a frame

@dataclass
class Sub:
    """One subframe.  `signal`: the target values before the wasted-bits shift (warm-up, verbatim and constant
    values must fit bps - wasted bits; predicted samples may be any i32).  `coefs[j]` multiplies s[t-1-j] (the first
    coefficient in the stream).  `params`: the Rice parameter of every partition, None for the cheapest; `method`
    None picks Rice2 only where a partition's cheapest parameter needs it.  The *_code fields and `escape` write
    raw values in place of the derived ones."""
    kind: str                       # "constant" | "verbatim" | "fixed" | "lpc"
    signal: list
    order: int = 0
    wasted: int = 0
    precision: int = 15
    shift: int = 0
    coefs: tuple = ()
    method: int | None = None
    porder: int = 0
    params: list | None = None
    pad: int = 0                    # the subframe's leading zero bit
    type_code: int | None = None
    wasted_zeros: int | None = None  # raw unary zeros after the wasted-bits flag
    precision_code: int | None = None
    shift_code: int | None = None   # raw 5-bit field
    method_code: int | None = None
    escape: tuple = ()              # partitions whose parameter is the escape code


@dataclass
class Frame:
    bps: int
    subs: list
    ca: int | None = None           # None: independent channels
    block_size: int | None = None   # None: the longest non-constant signal (1 if there is none)
    bs_code: int | None = None      # 6 / 7: an 8- / 16-bit block size after the number, whatever the size
    number: int = 0
    variable: bool = False
    sr_code: int = 9                # 44.1 kHz
    pad_fill: int = 0               # value of the pad bits before the CRC-16 (skipped unchecked)
    crc16_xor: int = 0
    truncate: int = 0               # bytes cut off the end

    @property
    def bs(self) -> int:
        if self.block_size is not None:
            return self.block_size
        return max([len(s.signal) for s in self.subs if s.kind != "constant"] or [1])


def _utf8(v: int) -> bytes:
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >= 1 << (5 * n + 1):
        n += 1
    out = [((0xFF << (8 - n)) & 0xFF) | (v >> (6 * (n - 1)))]
    out += [0x80 | ((v >> (6 * i)) & 0x3F) for i in reversed(range(n - 1))]
    return bytes(out)


def _bs_code(bs: int) -> tuple[int, bytes]:
    if bs == 192:
        return 1, b""
    for c in range(2, 6):
        if bs == 576 << (c - 2):
            return c, b""
    for c in range(8, 16):
        if bs == 256 << (c - 8):
            return c, b""
    if bs <= 256:
        return 6, bytes([bs - 1])
    return 7, (bs - 1).to_bytes(2, "big")


def sub_bits(f: Frame, ch: int) -> int:
    """Coded width of channel `ch` (one more for a side channel)."""
    return f.bps + (1 if (f.ca == 9 and ch == 0) or (f.ca in (8, 10) and ch == 1) else 0)


def zigzag(r: int) -> int:
    return (2 * r if r >= 0 else -2 * r - 1) & M32


def residuals(s: Sub) -> list[int]:
    x, n = s.signal, s.order
    if s.kind == "fixed":
        c = FIXED[n]
        out = []
        for t in range(n, len(x)):
            pred = 0
            for j, cj in enumerate(c):
                pred = i32(pred + i32(cj * x[t - 1 - j]))
            out.append(i32(x[t] - pred))
        return out
    return [i32(x[t] - (sum(c * x[t - 1 - j] for j, c in enumerate(s.coefs)) >> s.shift)) for t in range(n, len(x))]


def _cheapest(us: list[int], kmax: int) -> int:
    if not us:
        return 0
    best, bk = None, 0
    for k in range(kmax + 1):
        cost = sum((u >> k) + 1 + k for u in us)
        if best is None or cost < best:
            best, bk = cost, k
    return bk


def _write_sub(w: BitWriter, s: Sub, bits: int, bs: int, code_starts: list):
    w.put(s.pad, 1)
    order = s.order
    code = s.type_code
    if code is None:
        code = {"constant": 0, "verbatim": 1, "fixed": 8 | order, "lpc": 32 | ((order - 1) & 31)}[s.kind]
    w.put(code, 6)
    if s.wasted_zeros is not None:
        w.put(1, 1)
        w.unary(s.wasted_zeros)
    elif s.wasted:
        w.put(1, 1)
        w.unary(s.wasted - 1)
    else:
        w.put(0, 1)
    sb = bits - s.wasted
    if sb <= 0:
        return  # no non-wasted bits: the reference stops here
    if s.kind == "constant":
        w.put_signed(s.signal[0], sb)
        return
    if s.kind == "verbatim":
        for v in s.signal:
            w.put_signed(v, sb)
        return
    for v in s.signal[:order]:
        w.put_signed(v, sb)
    if s.kind == "lpc":
        w.put(s.precision - 1 if s.precision_code is None else s.precision_code, 4)
        if s.shift_code is not None:
            w.put(s.shift_code, 5)
        else:
            w.put_signed(s.shift, 5)
        for c in s.coefs:
            w.put_signed(c, s.precision)
    res = [zigzag(r) for r in residuals(s)]
    n_part = 1 << s.porder
    per = bs >> s.porder
    parts = []
    at = 0
    for p in range(n_part):
        n = max(0, per - order) if p == 0 else per
        parts.append(res[at:at + n])
        at += n
    ks = [s.params[p] if s.params is not None and s.params[p] is not None else None for p in range(n_part)]
    method = s.method
    if method is None:
        method = 1 if any(k is None and _cheapest(us, 30) > 14 or (k or 0) > 14 for k, us in zip(ks, parts)) else 0
    w.put(method if s.method_code is None else s.method_code, 2)
    w.put(s.porder, 4)
    kmax = 14 if method == 0 else 30
    pbits = 4 if method == 0 else 5
    for p, us in enumerate(parts):
        if p in s.escape:  # followed by the codes as if the escape were an ordinary parameter
            k = RICE_ESCAPE[method]
        else:
            k = ks[p] if ks[p] is not None else _cheapest(us, kmax)
        w.put(k, pbits)
        for u in us:
            code_starts.append(len(w))
            w.unary(u >> k)
            w.put(u & ((1 << k) - 1), k)


def write(f: Frame) -> tuple[bytes, dict]:
    """The frame's bytes and facts about them: pad bits, the bit position of every Rice code (from the frame's
    first byte), the header length."""
    bs = f.bs
    ca = f.ca if f.ca is not None else len(f.subs) - 1
    w = BitWriter()
    w.put(0xFFF8 | int(f.variable), 16)
    code, bs_extra = _bs_code(bs)
    if f.bs_code is not None:
        code, bs_extra = f.bs_code, (bs - 1).to_bytes(f.bs_code - 5, "big")
    w.put(code, 4)
    w.put(f.sr_code, 4)
    w.put(ca, 4)
    w.put(BPS_CODE[f.bps], 3)
    w.put(0, 1)
    head = w.to_bytes()[0] + _utf8(f.number) + bs_extra
    head += bytes([crc8(head)])
    w = BitWriter()
    for b in head:
        w.put(b, 8)
    starts: list = []
    for ch, s in enumerate(f.subs):
        _write_sub(w, s, sub_bits(f, ch), bs, starts)
    body, pad = w.to_bytes(f.pad_fill)
    data = body + (crc16(body) ^ f.crc16_xor).to_bytes(2, "big")
    if f.truncate:
        data = data[:-f.truncate]
    return data, dict(pad=pad, code_starts=starts, header_len=len(head))


def expected_pcm(f: Frame) -> np.ndarray:
    """Planar i32 output by construction."""
    bs = f.bs
    ch = [[i32(v << s.wasted) for v in (s.signal * bs if s.kind == "constant" else s.signal)][:bs] for s in f.subs]
    if f.ca == 8:
        ch = [ch[0], [i32(a - b) for a, b in zip(ch[0], ch[1])]]
    elif f.ca == 9:
        ch = [[i32(a + b) for a, b in zip(ch[0], ch[1])], ch[1]]
    elif f.ca == 10:
        left, right = [], []
        for m, s in zip(ch[0], ch[1]):
            m2 = i32(i32(m << 1) | (s & 1))
            left.append(i32(m2 + s) >> 1)
            right.append(i32(m2 - s) >> 1)
        ch = [left, right]
    return np.array(ch, np.int64).astype(np.int32).reshape(-1)


# --------------------------------------------------------------------------- catalogue entries

@dataclass
class Entry:
    """One frame: `status` is the reference's verdict, `pcm` the planar output by construction (also given for a
    frame whose only fault is its CRC-16, which is what a decoder that skips the check produces); `channel` the
    subframe an error sits in (None for a frame-level one); `tags`: which groups of tests the entry belongs to."""
    name: str
    data: bytes
    status: int
    pcm: np.ndarray | None
    channel: int | None = None
    tags: frozenset = frozenset()
    frame: Frame | None = None
    info: dict = field(default_factory=dict)

    @property
    def n_channels(self) -> int:
        return len(self.frame.subs)

    @property
    def in_width(self) -> bool:
        """Every subframe signal after the wasted-bits shift lies inside its coded width (fastpath.keeps_width)."""
        f = self.frame
        for ch, s in enumerate(f.subs):
            b = sub_bits(f, ch)
            vals = [i32(v << s.wasted) for v in s.signal]
            if min(vals) < -(1 << (b - 1)) or max(vals) >= 1 << (b - 1):
                return False
        return True


def entry(name, f: Frame, status=OK, channel=None, tags=()) -> Entry:
    data, info = write(f)
    pcm = expected_pcm(f) if status in (OK, CRC_MISMATCH) else None
    return Entry(name, data, status, pcm, channel, frozenset(tags), f, info)


def lo(b):
    return -(1 << (b - 1))


def hi(b):
    return (1 << (b - 1)) - 1


def extremes(b: int, n: int, seed: int = 0) -> list[int]:
    """n samples at the two extremes of b bits, in a pattern that holds runs of both and every transition."""
    rng = np.random.default_rng(seed)
    base = [lo(b), hi(b), hi(b), lo(b), lo(b), lo(b), hi(b), hi(b), hi(b), hi(b)]
    return (base + [hi(b) if x else lo(b) for x in rng.integers(0, 2, max(0, n - len(base)))])[:n]


def lpc_full(order: int, precision: int = 15) -> tuple:
    """Coefficients at the extremes of `precision` bits, alternating in sign."""
    return tuple((hi(precision) if j % 2 else lo(precision)) for j in range(order))


def predictors(b: int, sig: list[int]) -> dict:
    """Each subframe kind holding `sig` (b-bit values)."""
    out = {"constant": Sub("constant", [sig[0]]), "verbatim": Sub("verbatim", sig)}
    for n in range(5):
        out[f"fixed{n}"] = Sub("fixed", sig, order=n, porder=1 if len(sig) % 2 == 0 and n <= len(sig) // 2 else 0)
    out["lpc8"] = Sub("lpc", sig, order=8, precision=15, shift=14, coefs=lpc_full(8))
    out["lpc32-p1"] = Sub("lpc", sig, order=32, precision=1, shift=0, coefs=(-1,) * 32)
    return out


def stereo(bps: int, ca: int, left: list, right: list, kind: str, wasted: int = 0) -> Frame:
    """Left/right targets coded with `ca` (1 independent, 8 left/side, 9 side/right, 10 mid/side), both subframes
    of predictor `kind` (a key of predictors())."""
    side = [a - b for a, b in zip(left, right)]
    mid = [(a + b) >> 1 for a, b in zip(left, right)]
    chans = {1: (left, right), 8: (left, side), 9: (side, right), 10: (mid, side)}[ca]
    subs = []
    for c in chans:
        if kind == "constant" and len(set(c)) != 1:
            s = Sub("verbatim", list(c))
        else:
            s = replace(predictors(bps + 1, list(c))[kind], signal=list(c))
        subs.append(replace(s, wasted=wasted))
    return Frame(bps, subs, ca=ca, block_size=len(left))


# --------------------------------------------------------------------------- the catalogue

WIDTHS = (8, 12, 16, 20, 24)
CA_NAMES = {0: "mono", 1: "indep", 8: "left-side", 9: "side-right", 10: "mid-side"}


def _full_scale() -> list[Entry]:
    out = []
    for b in WIDTHS:
        left = extremes(b, 64, seed=b)
        right = extremes(b, 64, seed=b + 100)
        for kind in ("constant", "verbatim", "fixed0", "fixed1", "fixed2", "fixed3", "fixed4", "lpc8", "lpc32-p1"):
            for ca in (0, 1, 8, 9, 10):
                if ca == 0:
                    sig = [left[0]] * 64 if kind == "constant" else left
                    f = Frame(b, [replace(predictors(b, sig)[kind], signal=sig)], block_size=64)
                else:
                    r = list(left) if kind == "constant" else right
                    f = stereo(b, ca, [left[0]] * 64 if kind == "constant" else left,
                               [r[0]] * 64 if kind == "constant" else r, kind)
                out.append(entry(f"full-scale/{b}bit/{CA_NAMES[ca]}/{kind}", f, tags={"full-scale", "in-width"}))
        # a side channel at both extremes of its b + 1 bits (-2^b needs a right channel one past 2^(b-1) - 1)
        side = [lo(b + 1), hi(b + 1)] * 16
        left = [lo(b), hi(b)] * 16
        f = Frame(b, [Sub("verbatim", left), Sub("fixed", side, order=2)], ca=8)
        out.append(entry(f"full-scale/{b}bit/side-at-both-extremes", f, tags={"full-scale", "in-width"}))
    # a whole warp of these reaches the straight-line flushes: 16-bit stereo, independent and mid/side, 256 samples
    for ca in (1, 10):
        left, right = extremes(16, 256, seed=1), extremes(16, 256, seed=2)
        for kind in ("fixed2", "lpc8"):
            f = stereo(16, ca, left, right, kind)
            out.append(entry(f"full-scale/16bit/{CA_NAMES[ca]}/{kind}/256", f, tags={"full-scale", "in-width", "flush"}))
    return out


def _acc_boundary() -> list[Entry]:
    """sum|coef| << (b-1) just below, on and just above 2^31, with negative coefficients and every sample at -2^(b-1):
    each product is positive, so the sum is +absum * 2^(b-1), which an i32 accumulator wraps from 2^31 on."""
    out = []
    for b in WIDTHS:
        for side in (False, True):
            bits = b + side
            for order in (1, 8, 12, 32):
                for delta in (-1, 0, 1):
                    absum = (1 << (32 - bits)) + delta
                    if absum > order * (1 << 14):
                        continue  # not reachable with 15-bit coefficients
                    q, rem = divmod(absum, order)
                    coefs = tuple(-(q + (j < rem)) for j in range(order))
                    shift = min(15, max(0, absum.bit_length() - 1))
                    n = 64
                    sig = [lo(bits)] * n
                    sub = Sub("lpc", sig, order=order, precision=15, shift=shift, coefs=coefs, porder=0)
                    if side:
                        f = Frame(b, [Sub("verbatim", [lo(b)] * n), sub], ca=8)
                    else:
                        f = Frame(b, [sub])
                    tag = {-1: "below", 0: "on", 1: "above"}[delta]
                    out.append(entry(f"acc-boundary/{b}bit{'/side' if side else ''}/order{order}/{tag}", f,
                                     tags={"acc-boundary", "in-width"}))
    return out


def _mid_side_bound() -> list[Entry]:
    out = []
    n = 32
    for wasted in (0, 2):
        for d in (-1, 0, 1):  # (with wasted bits: one step of 2^wasted either side of 2^29)
            v = (1 << (29 - wasted)) + d
            mid = [v, -v, 3, -v, v] + [7] * (n - 5)
            side = [1, -1, v, 2, -3] + [5] * (n - 5)
            f = Frame(16, [Sub("fixed", mid, order=0, wasted=wasted), Sub("fixed", side, order=0, wasted=wasted)],
                      ca=10)
            out.append(entry(f"ms-bound/(2^{29 - wasted}{d:+d})<<{wasted}", f, tags={"ms-bound"}))
    # |M|, |S| < 2^30 with 2|M| + |S| >= 2^31: the wrapping intermediate (m << 1 | s & 1) +- s differs from
    # M + (S >> 1) + (S & 1)
    for m, s in (((1 << 30) - 1, (1 << 30) - 1), (-(1 << 30), -(1 << 30) + 1), ((1 << 30) - 3, 5),
                 (-(1 << 30) + 1, (1 << 29) + 7), ((3 << 28) + 1, -(1 << 29) - 1)):
        mid = [m, -m, m, 0] * 8
        side = [s, s, -s, s] * 8
        f = Frame(24, [Sub("fixed", mid, order=0), Sub("fixed", side, order=0)], ca=10)
        out.append(entry(f"ms-wrap/{m}/{s}", f, tags={"ms-bound", "ms-wrap"}))
    return out


def _coefs_shift() -> list[Entry]:
    out = []
    b = 16
    sig = extremes(b, 48, seed=5)
    for p in (1, 15):
        for c in (lo(p), hi(p)):
            if c == 0:
                continue
            for order in (1, 12, 32):
                for shift in (0, 15):
                    f = Frame(b, [Sub("lpc", sig, order=order, precision=p, shift=shift, coefs=(c,) * order)])
                    out.append(entry(f"coefs/p{p}/c{c}/order{order}/shift{shift}", f, tags={"coefs", "in-width"}))
    # large coefficients with shift 0: the prediction wraps i32 (the residuals absorb it)
    f = Frame(24, [Sub("lpc", extremes(24, 48, seed=6), order=4, precision=15, shift=0, coefs=(lo(15),) * 4)])
    out.append(entry("coefs/p15-shift0-order4/24bit", f, tags={"coefs", "in-width"}))
    return out


def _rice() -> list[Entry]:
    out = []
    b = 16
    # parameters at the top of their ranges
    sig = [lo(8), hi(8)] * 32
    out.append(entry("rice/k0-extremes", Frame(8, [Sub("fixed", sig, order=0, params=[0])]), tags={"rice", "in-width"}))
    sig = [lo(b), hi(b)] * 32
    out.append(entry("rice/k14-extremes", Frame(b, [Sub("fixed", sig, order=1, params=[14])]), tags={"rice", "in-width"}))
    big = [-(1 << 31), (1 << 31) - 1, -(1 << 31), -1, 0, (1 << 31) - 1] * 6
    for k in (30, 29):
        f = Frame(b, [Sub("fixed", big, order=0, method=1, params=[k])])
        out.append(entry(f"rice2/k{k}-residuals-at-2^31", f, tags={"rice"}))
    # a code of exactly 32 bits: k = 0, q = 31 (u = 31: residual -16)
    one = [0] * 20 + [-16] + [0] * 11
    out.append(entry("rice/code-32-bits", Frame(b, [Sub("fixed", one, order=0, params=[0])]), tags={"rice", "in-width"}))
    # pairs of codes 32 and 33 bits long together, at k <= 6, in a stepped channel and in the last channel
    for k in (0, 3, 6):
        q = (32 - 2 * (k + 1)) // 2
        u32 = [(q << k) | (i % (1 << k) if k else 0) for i in range(64)]                    # every pair: 32 bits
        u33 = [((q + (i & 1)) << k) | (i % (1 << k) if k else 0) for i in range(64)]        # every pair: 33 bits
        for tag, us in (("32", u32), ("33", u33)):
            r = [(u >> 1) ^ -(u & 1) for u in us]
            code = Sub("fixed", r, order=0, params=[k])
            filler = Sub("fixed", [(-1) ** i * (i % 7) for i in range(64)], order=1)
            for pos in ("first", "last"):
                subs = [code, filler, filler] if pos == "first" else [filler, filler, code]
                out.append(entry(f"rice/pairs-{tag}-bits/k{k}/{pos}-of-3", Frame(b, subs), tags={"rice", "in-width"}))
    # long unary runs: 1023..1025 bits (the 128-byte decode ring), 2047..2049 (the 256-byte index ring)
    for q in (1023, 1024, 1025, 2047, 2048, 2049):
        r = (q >> 1) ^ -(q & 1)
        sig = [3, -2, 1] + [r] + [0, 1, -1] * 9 + [r]
        for nch in (1, 2):
            subs = [Sub("fixed", sig, order=0, params=[0])] * nch
            out.append(entry(f"rice/unary-{q}/{nch}ch", Frame(b, subs), tags={"rice", "long-unary", "in-width"}))
    # runs that end 1 before, on and 1 after the warp path's window limit (4064 - start bit mod 128), at a frame
    # placed on a 16-byte boundary
    for d in (-1, 0, 1):
        sig = [1, 2] + [0] * 30
        f = Frame(b, [Sub("fixed", sig, order=0, params=[0])])
        _, info = write(f)
        p = info["code_starts"][2]
        q = 4064 - (p & 127) + d
        sig[2] = (q >> 1) ^ -(q & 1)
        out.append(entry(f"rice/warp-window{d:+d}", f, tags={"rice", "long-unary", "warp-window", "in-width"}))
    # escape parameters: first, a middle and the last partition, and an empty first one
    sig = [(-1) ** i * (i % 11) for i in range(64)]
    for method in (0, 1):
        for p in (0, 2, 3):
            f = Frame(b, [Sub("fixed", sig, order=1, porder=2, method=method, escape=(p,))])
            out.append(entry(f"rice/escape/method{method}/part{p}", f, ESCAPE, 0, tags={"rice", "error"}))
        f = Frame(b, [Sub("fixed", sig[:16], order=4, porder=2, method=method, escape=(0,))])
        out.append(entry(f"rice/escape/method{method}/empty-part", f, ESCAPE, 0, tags={"rice", "error"}))
    # partitions of every length 1..9: a partition boundary at every position of a group of eight
    for per in range(1, 10):
        for order in (0, 1):
            if order > per:
                continue
            sig = [(-1) ** i * ((i * 7) % 23) for i in range(per * 8)]
            f = Frame(b, [Sub("fixed", sig, order=order, porder=3)])
            out.append(entry(f"rice/partition-length-{per}/order{order}", f, tags={"rice", "in-width"}))
    # an empty first partition, still carrying a parameter
    sig = extremes(b, 32, seed=9)
    f = Frame(b, [Sub("lpc", sig, order=8, precision=12, shift=11, coefs=(300, -120, 50, -20, 9, -4, 2, -1), porder=2)])
    out.append(entry("rice/empty-first-partition/lpc8", f, tags={"rice", "in-width"}))
    f = Frame(b, [Sub("fixed", sig[:8], order=4, porder=1)])
    out.append(entry("rice/empty-first-partition/fixed4", f, tags={"rice", "in-width"}))
    # partition order 15 at block size 32768: one residual per partition
    sig = [(i * 37) % 200 - 100 for i in range(32768)]
    f = Frame(b, [Sub("fixed", sig, order=1, porder=15)])
    out.append(entry("rice/partition-order-15", f, tags={"rice", "in-width", "large"}))
    return out


def _degenerate() -> list[Entry]:
    out = []
    b = 16
    out.append(entry("shape/block-size-1/verbatim", Frame(b, [Sub("verbatim", [lo(b)]), Sub("verbatim", [hi(b)])]),
                     tags={"shape", "in-width"}))
    out.append(entry("shape/block-size-1/fixed1", Frame(b, [Sub("fixed", [hi(b)], order=1)]), tags={"shape", "in-width"}))
    out.append(entry("shape/block-size-1/constant-ms",
                     Frame(b, [Sub("constant", [lo(b)]), Sub("constant", [hi(b + 1)])], ca=10),
                     tags={"shape", "in-width"}))
    sig32 = extremes(b, 32, seed=3)
    out.append(entry("shape/lpc32-at-block-16", Frame(b, [Sub("lpc", sig32[:16] + [0] * 16, order=32, coefs=(1,) * 32)],
                                                        block_size=16), LPC_GT_BLOCK, 0, tags={"shape", "error"}))
    out.append(entry("shape/lpc32-at-block-32-no-residuals",
                     Frame(b, [Sub("lpc", sig32, order=32, precision=15, shift=15, coefs=lpc_full(32))]),
                     tags={"shape", "in-width"}))
    out.append(entry("shape/fixed4-at-block-4", Frame(b, [Sub("fixed", sig32[:4], order=4)]), tags={"shape", "in-width"}))
    out.append(entry("shape/fixed4-at-block-3", Frame(b, [Sub("fixed", sig32[:4], order=4)], block_size=3),
                     FIXED_GT_BLOCK, 0, tags={"shape", "error"}))
    sig = [((i * 2654435761) >> 7) % 60001 - 30000 for i in range(65535)]
    out.append(entry("shape/block-size-65535", Frame(b, [Sub("fixed", sig, order=2)]), tags={"shape", "in-width", "large"}))
    # wasted bits at bps - 1 (one bit left) and, on a side channel, at bps
    for bb in (8, 16, 24):
        one = [0, -1, -1, 0] * 8
        out.append(entry(f"shape/wasted-{bb - 1}-of-{bb}", Frame(bb, [Sub("verbatim", one, wasted=bb - 1)]),
                         tags={"shape", "in-width"}))
        f = Frame(bb, [Sub("fixed", [0] * 32, order=0, wasted=bb - 1), Sub("verbatim", one, wasted=bb)], ca=8)
        out.append(entry(f"shape/side-wasted-{bb}-of-{bb + 1}", f, tags={"shape", "in-width"}))
    # pad bits before the CRC-16: none, and seven (set to one: they are skipped unchecked)
    out.append(entry("shape/no-pad-bits", Frame(16, [Sub("verbatim", [hi(15)], wasted=1)]), tags={"shape", "in-width"}))
    out.append(entry("shape/seven-pad-bits", Frame(16, [Sub("verbatim", extremes(15, 8), wasted=1)], pad_fill=1),
                     tags={"shape", "in-width"}))
    # variable blocking with a 7-byte sample number, and 8- and 16-bit block-size codes at their limits
    out.append(entry("shape/variable-blocking", Frame(16, [Sub("fixed", sig32, order=3)], variable=True,
                                                      number=(1 << 36) - 32), tags={"shape", "in-width"}))
    out.append(entry("shape/block-size-256-8bit-code", Frame(16, [Sub("fixed", extremes(16, 256), order=2)], bs_code=6),
                     tags={"shape", "in-width"}))
    out.append(entry("shape/block-size-1-16bit-code", Frame(16, [Sub("verbatim", [lo(16)])], bs_code=7),
                     tags={"shape", "in-width"}))
    return out


def _filler(i: int, bps: int, n: int = 32) -> Sub:
    """A valid subframe of n samples, of one of four kinds."""
    sig = extremes(bps, n, seed=40 + i)
    po = 0 if n % 4 else 2
    subs = [Sub("constant", [hi(bps)]), Sub("verbatim", sig), Sub("fixed", sig, order=3, porder=po),
            Sub("lpc", sig, order=5, precision=9, shift=8, coefs=(200, -90, 40, -10, 3), porder=po // 2)]
    return subs[i % 4] if n >= 8 else subs[i % 2]


def _errors() -> list[Entry]:
    out = []
    b = 16
    sig = [(-1) ** i * (i % 13) for i in range(32)]
    mono = {
        PAD_BIT: Sub("fixed", sig, order=2, pad=1),
        WASTED_GT_31: Sub("fixed", sig, order=2, wasted_zeros=32),
        NO_NON_WASTED: Sub("verbatim", [0] * 32, wasted=b),
        RES_RESERVED: Sub("fixed", sig, order=2, method_code=2),
        PORDER_INVALID: Sub("fixed", sig[:31], order=2, porder=1, method_code=None),
        RES_INVALID: Sub("fixed", sig, order=3, porder=4),  # 2 samples per partition < order 3
        ESCAPE: Sub("fixed", sig, order=2, porder=1, escape=(1,)),
        PRECISION_INVALID: Sub("lpc", sig, order=2, coefs=(1, 1), precision_code=15),
        NEGATIVE_SHIFT: Sub("lpc", sig, order=2, coefs=(1, 1), shift_code=0b11111),
    }
    for status, s in mono.items():
        out.append(entry(f"error/{status}/mono", Frame(b, [s]), status, 0, tags={"error"}))
    out.append(entry("error/15/method3", Frame(b, [Sub("fixed", sig, order=2, method_code=3)]), RES_RESERVED, 0,
                     tags={"error"}))
    out.append(entry("error/13/wasted-zeros-31", Frame(b, [Sub("fixed", sig, order=2, wasted_zeros=31)]), WASTED_GT_31,
                     0, tags={"error"}))
    out.append(entry("error/14/wasted-24-of-24", Frame(24, [Sub("verbatim", [0] * 32, wasted=24)]), NO_NON_WASTED, 0,
                     tags={"error"}))
    for code in (2, 3, 4, 5, 6, 7, 13, 14, 15) + tuple(range(16, 32)):
        out.append(entry(f"error/12/type-code-{code}", Frame(b, [Sub("fixed", sig, order=2, type_code=code)]),
                         SUB_RESERVED, 0, tags={"error"}))
    # each subframe error in channel 0, a middle channel and the last channel of 3- and 8-channel frames
    placed = {**mono, SUB_RESERVED: Sub("fixed", sig, order=2, type_code=0b010000),
              FIXED_GT_BLOCK: None, LPC_GT_BLOCK: None}
    for status in sorted(placed):
        for nch in (3, 8):
            for ch in (0, nch // 2, nch - 1):
                bs = {FIXED_GT_BLOCK: 3, LPC_GT_BLOCK: 3, PORDER_INVALID: 31}.get(status, 32)
                subs = [_filler(i, b, bs) for i in range(nch)]
                subs[ch] = {FIXED_GT_BLOCK: Sub("fixed", [1, 2, 3, 4], order=4),
                            LPC_GT_BLOCK: Sub("lpc", [1, 2, 3, 4, 5], order=5, coefs=(1,) * 5)}.get(status, placed[status])
                f = Frame(b, subs, block_size=bs)
                out.append(entry(f"error/{status}/{nch}ch/channel{ch}", f, status, ch, tags={"error", "placed"}))
    # frame-level: truncation inside the last Rice code, and a CRC-16 mismatch
    for nch in (1, 3, 8):
        subs = [_filler(i, b) for i in range(nch - 1)] + [Sub("fixed", [0] * 31 + [-600], order=0, params=[0])]
        out.append(entry(f"error/2/truncated-in-last-code/{nch}ch", Frame(b, subs, truncate=5), EOF_ERR, None,
                         tags={"error"}))
        out.append(entry(f"error/23/crc16/{nch}ch", Frame(b, subs, crc16_xor=0x0100), CRC_MISMATCH, None,
                         tags={"error", "crc"}))
    return out


def _multichannel() -> list[Entry]:
    """3, 5, 7 and 8 channels, each channel a different edge."""
    out = []
    b = 16
    n = 64
    edges = [
        Sub("verbatim", extremes(b, n, seed=71)),
        Sub("lpc", extremes(b, n, seed=72), order=32, precision=15, shift=15, coefs=lpc_full(32), porder=1),
        Sub("fixed", [0] * 20 + [-16] + [0] * 43, order=0, params=[0]),                                # 32-bit code
        Sub("fixed", [3] + [(1023 >> 1) ^ -1] + [0] * (n - 2), order=0, params=[0]),                    # 1023 zeros
        Sub("verbatim", [0, -1] * (n // 2), wasted=b - 1),
        Sub("fixed", extremes(b, n, seed=73), order=4, porder=3),
        Sub("lpc", [lo(b)] * n, order=12, precision=15, shift=12, coefs=(-((1 << 16) // 12 + 1),) * 12),  # absum >= 2^16
        Sub("constant", [lo(b)]),
    ]
    for nch in (3, 5, 7, 8):
        subs = [edges[(i * 3 + nch) % len(edges)] for i in range(nch)]
        out.append(entry(f"multichannel/{nch}ch", Frame(b, subs), tags={"multichannel", "in-width"}))
    return out


CATALOGUE: list[Entry] = (_full_scale() + _acc_boundary() + _mid_side_bound() + _coefs_shift() + _rice()
                          + _degenerate() + _errors() + _multichannel())
BY_NAME = {e.name: e for e in CATALOGUE}
assert len(BY_NAME) == len(CATALOGUE), "entry names must be unique"


# --------------------------------------------------------------------------- batches

def batch(entries: list[Entry], gaps=None):
    """One byte buffer holding the entries' frames (frame i preceded by gaps[i] filler bytes).  Returns data, offsets,
    lengths, and the expected planar PCM laid out at the out_offsets descs_from_offsets gives these frames (an
    entry without PCM leaves its span at 0)."""
    parts, offs, at = [], [], 0
    for i, e in enumerate(entries):
        g = 0 if gaps is None else int(gaps[i])
        parts.append(bytes([0xA5]) * g)
        at += g
        offs.append(at)
        parts.append(e.data)
        at += len(e.data)
    data = np.frombuffer(b"".join(parts), np.uint8).copy()
    lens = np.array([len(e.data) for e in entries], np.uint32)
    offs = np.array(offs, np.uint64)
    exp, o = [], 0
    out_offsets = []
    for e in entries:
        n = e.n_channels * e.frame.bs
        out_offsets.append(o)
        o += (n + 3) & ~3
    ref = np.zeros(max(1, o), np.int32)
    for e, oo in zip(entries, out_offsets):
        if e.pcm is not None:
            ref[oo:oo + e.pcm.size] = e.pcm
    return data, offs, lens, ref
