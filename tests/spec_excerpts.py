"""The excerpt plan of crop and packed batches, restated in plain Python, and checkers of whole device outputs against
it (test helper, no tests here).

From include/claxon_b200.h and DESIGN §3.6, not from the kernels:

    request_ok(file, reserved, offset, length, n_files)   a request the planner reads at all
    excerpt_length(offset, length, N)                      n_b, or -1 for an offset past N
    length_at(N, r, R)                                     N_t = ceil(N n / o) at target rate R (N for r == R)
    packed_plan(files, offsets, lengths, Ns, T, count, max_excerpts)
                                                           starts, lengths, statuses, the error word and the end column
    crop_plan(files, offsets, L, Ns)                       lengths, statuses and the error word of a crop batch
    mel_plan(plan, n_fft, hop, center)                     F_b and the frame starts of a mel packed batch

A packed batch's start_b is the exclusive scan of round_up_4(n_b) over the valid excerpts (n_b = 0 for an invalid one),
whether they fit or not; excerpt b fits when start_b + n_b <= T.  An invalid or non-fitting excerpt has length 0 and
status CLX_ERR_INVALID_ARGUMENT (90); excerpts past `count` are unused (length 0, status 0).  The error word is the
smallest (kind << 62) | (b << 32) | status over the failed excerpts, kind 0 for a planner failure, all ones for none.
A call's end column is the furthest min(start_b + round_up_4(n_b), T) of an excerpt that fits and has samples: what the
next call's zero pass clears back to.

The checkers build the full expected [C, T] (or [B, C, L], or [C, n_mels, T_f]) tensor from per-excerpt references, every
element outside an excerpt exactly 0, and assert the device output against it:

    expected_packed(plan, files, offsets, pcm, C, T)       the integer / float32 rows of load() of each file
    expected_crops(plan, files, offsets, pcm, C, L)
    expected_resampled(plan, files, offsets, refs, C, T)   float64 FIR reference and bound (tests/spec_signal.py)
    check_exact(dev, want)                                  bit for bit, as int32 words
    check_bound(dev, ref, bound)                            |dev - ref| <= bound everywhere (0 outside excerpts)
    check_plan(plan, starts, lengths, status, error)        the bookkeeping of one call
    per_feature_packed(y, x, starts, frames)                normalised packed features within an ulp of the map of x
    per_feature_crops(y, x, valid)                          the same for crop features
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from tests import spec_mel_norm as MN
from tests import spec_resample as SR

ERR_INVALID = 90
NO_ERROR = (1 << 64) - 1


def r4(x: int) -> int:
    return (x + 3) & ~3


def request_ok(file: int, reserved: int, offset: int, length: int, n_files: int) -> bool:
    return reserved == 0 and 0 <= file < n_files and offset >= 0 and length != 0 and length >= -1


def excerpt_length(offset: int, length: int, N: int) -> int:
    """min(length, N - offset) (N - offset for length -1); -1 for an offset past N."""
    if offset > N:
        return -1
    rest = N - offset
    return rest if length == -1 or length > rest else length


def length_at(N: int, r: int, R: int | None) -> int:
    return N if R is None else SR.out_len(N, r, R)


def split_file(f: int) -> tuple[int, int]:
    """A files-column value as the request's (file, reserved) pair: the low and high 32 bits."""
    f &= (1 << 64) - 1
    return f & 0xffffffff, f >> 32


def error_word(failed) -> int:
    """The smallest (kind << 62) | (b << 32) | status of (kind, b, status) triples; NO_ERROR for none."""
    return min(((k << 62) | (b << 32) | (s & 0xffffffff) for k, b, s in failed), default=NO_ERROR)


@dataclass
class Plan:
    starts: list      # start_b (column, or frame column for mel_plan)
    lengths: list     # n_b as the batch reports it: 0 for an invalid, non-fitting or unused excerpt
    status: list      # 0 or ERR_INVALID
    error: int        # the expected error word, unsigned
    end: int = 0      # the call's end column (packed batches)

    @property
    def fits(self) -> list:
        return [s == 0 for s in self.status]


def packed_plan(files, offsets, lengths, Ns, T: int, count: int | None = None, max_excerpts: int | None = None) -> Plan:
    """The plan of a packed call of the first `count` requests (all of them by default); Ns each file's length at the
    batch's rate.  With max_excerpts (the batch's), lengths and statuses also cover the unused excerpts count ..
    max_excerpts - 1: length 0 and status 0 whatever an earlier call left there; starts cover the used ones only."""
    n = len(files) if count is None else count
    starts, lens, status = [], [], []
    at = end = 0
    for b in range(n):
        f, res = split_file(int(files[b]))
        o, ln = int(offsets[b]), int(lengths[b])
        nb = excerpt_length(o, ln, Ns[f]) if request_ok(f, res, o, ln, len(Ns)) else -1
        starts.append(at)
        if nb < 0:
            lens.append(0), status.append(ERR_INVALID)
            continue
        if at + nb > T:
            lens.append(0), status.append(ERR_INVALID)
        else:
            lens.append(nb), status.append(0)
            if nb:
                end = max(end, min(at + r4(nb), T))
        at += r4(nb)
    err = error_word((0, b, s) for b, s in enumerate(status) if s)
    if max_excerpts is not None:
        assert max_excerpts >= n
        lens += [0] * (max_excerpts - n)
        status += [0] * (max_excerpts - n)
    return Plan(starts, lens, status, err, end)


def crop_plan(files, offsets, L: int, Ns) -> Plan:
    """A crop batch: crop b is request (file, offset, L); every valid crop fits, starts are b * C * L."""
    lens, status = [], []
    for f, o in zip(files, offsets):
        f, res = split_file(int(f))
        nb = excerpt_length(int(o), L, Ns[f]) if request_ok(f, res, int(o), L, len(Ns)) else -1
        lens.append(max(nb, 0)), status.append(0 if nb >= 0 else ERR_INVALID)
    err = error_word((0, b, s) for b, s in enumerate(status) if s)
    return Plan([0] * len(lens), lens, status, err)


def mel_frame_count(n: int, n_fft: int, hop: int, center: bool) -> int:
    if center:
        return 1 + n // hop if n > n_fft // 2 else 0
    return 1 + (n - n_fft) // hop if n >= n_fft else 0


def mel_plan(plan: Plan, n_fft: int, hop: int, center: bool = True) -> Plan:
    """The frame layout of a mel packed batch over `plan`'s excerpts: F_b of n_b, starts the scan of round_up_4(F_b)."""
    starts, frames, at = [], [], 0
    for nb in plan.lengths:
        F = mel_frame_count(nb, n_fft, hop, center)
        starts.append(at), frames.append(F)
        at += r4(F)
    return Plan(starts, frames, plan.status, plan.error, at)


# --------------------------------------------------------------------------- expected tensors and checks

def expected_packed(plan: Plan, files, offsets, pcm, C: int, T: int, dtype=np.int32) -> np.ndarray:
    """[C, T]: excerpt b's rows pcm[f][:, o : o + n_b] at columns from start_b, 0 everywhere else."""
    out = np.zeros((C, T), dtype)
    for b, (s, n) in enumerate(zip(plan.starts, plan.lengths)):
        if n:
            x = pcm[split_file(int(files[b]))[0]]
            o = int(offsets[b])
            out[:x.shape[0], s:s + n] = x[:, o:o + n]
    return out


def expected_crops(plan: Plan, files, offsets, pcm, C: int, L: int, dtype=np.int32) -> np.ndarray:
    """[B, C, L]: crop b's rows pcm[f][:, o : o + n_b], 0 past n_b and on rows its file lacks."""
    out = np.zeros((len(plan.lengths), C, L), dtype)
    for b, n in enumerate(plan.lengths):
        if n:
            x = pcm[split_file(int(files[b]))[0]]
            o = int(offsets[b])
            out[b, :x.shape[0], :n] = x[:, o:o + n]
    return out


def expected_resampled(plan: Plan, files, offsets, refs, C: int, T: int):
    """(ref, bound) [C, T] of a resampled packed call: refs[f] = (ref, bound) of file f's whole signal at R
    (spec_signal.fir_ref_bound), sliced per excerpt; 0 and 0 (so exactly 0 required) everywhere else."""
    ref, bound = np.zeros((C, T)), np.zeros((C, T))
    for b, (s, n) in enumerate(zip(plan.starts, plan.lengths)):
        if n:
            r, bd = refs[split_file(int(files[b]))[0]]
            o = int(offsets[b])
            ref[:r.shape[0], s:s + n] = r[:, o:o + n]
            bound[:r.shape[0], s:s + n] = bd[:, o:o + n]
    return ref, bound


def check_exact(dev, want, what: str = ""):
    """dev and want bit for bit (as 32-bit words, so -0.0 and 0.0 differ)."""
    d = np.ascontiguousarray(dev).view(np.int32)
    w = np.ascontiguousarray(want).astype(np.asarray(dev).dtype).view(np.int32)
    assert d.shape == w.shape, (what, d.shape, w.shape)
    bad = d != w
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4].tolist())


def check_bound(dev, ref, bound, what: str = "") -> float:
    """|dev - ref| <= bound everywhere, exactly equal where the bound is 0; returns the worst ratio."""
    dev = np.asarray(dev, dtype=np.float64)
    err = np.abs(dev - ref)
    bad = err > bound
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4].tolist())
    return float((err / np.where(bound > 0, bound, 1.0)).max(initial=0.0))


def check_plan(plan: Plan, starts, lengths, status, error, what: str = ""):
    """One call's starts (packed batches; None to skip), lengths, statuses and error word against the plan."""
    n = len(plan.lengths)
    if starts is not None:
        starts = np.asarray(starts).tolist()
        assert starts == plan.starts, (what, "starts", first_diff(starts, plan.starts))
    lengths, status = np.asarray(lengths).tolist(), np.asarray(status).tolist()
    assert len(lengths) == n and len(status) == n, what
    assert lengths == plan.lengths, (what, "lengths", first_diff(lengths, plan.lengths))
    assert status == plan.status, (what, "status", first_diff(status, plan.status))
    err = int(error) & NO_ERROR
    assert err == plan.error, (what, "error word", hex(err), hex(plan.error))


def first_diff(a, b):
    i = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
    return i, a[i:i + 3], b[i:i + 3]


def ulp_ratio(dev, ref) -> float:
    """spec_mel_norm.within_ulp's assertion; returns the largest error in units of that ulp."""
    MN.within_ulp(dev, ref)
    dev = np.asarray(dev, dtype=np.float32)
    ulp = np.spacing(np.maximum(np.abs(dev), np.abs(np.asarray(ref).astype(np.float32)))).astype(np.float64)
    return float((np.abs(dev.astype(np.float64) - ref) / ulp).max(initial=0.0))


def per_feature_packed(y, x, starts, frames, chunk: int = 4096) -> float:
    """Asserts packed features y [C, n_mels, T_f] within one float32 ulp of spec_mel_norm's per-feature map of x (the
    same call's unnormalised features) over each excerpt's F_b frame columns, and exactly 0 everywhere else.  Excerpts
    of one frame count are mapped together, `chunk` of them at a time.  Returns the largest error in ulps."""
    y, x = np.asarray(y), np.asarray(x)
    starts, frames = np.asarray(starts, dtype=np.int64), np.asarray(frames, dtype=np.int64)
    covered = np.zeros(y.shape[-1], bool)
    worst = 0.0
    for F in np.unique(frames[frames > 0]):
        sel = np.flatnonzero(frames == F)
        for a in range(0, sel.size, chunk):
            cols = starts[sel[a:a + chunk]][:, None] + np.arange(F)[None, :]     # [k, F]
            seg = x[:, :, cols].astype(np.float64)                                 # [C, n_mels, k, F]
            mu, sigma = MN.stats(seg, int(F))
            worst = max(worst, ulp_ratio(y[:, :, cols], (seg - mu) / (sigma + MN.EPS)))
            covered[cols.ravel()] = True
    rest = y[:, :, ~covered]
    assert not rest.any(), ("outside the excerpts' frames", np.argwhere(rest != 0)[:4].tolist())
    return worst


def per_feature_crops(y, x, valid, chunk: int = 4096) -> float:
    """Asserts crop features y [B, C, n_mels, F] within one float32 ulp of spec_mel_norm's per-feature map of x over
    crop b's first valid[b] frames, and exactly 0 from there on; `chunk` crops at a time.  Returns the largest error in
    ulps."""
    worst = 0.0
    y, x, valid = np.asarray(y), np.asarray(x), np.asarray(valid)
    for a in range(0, len(valid), chunk):
        yc, xc, vc = y[a:a + chunk], x[a:a + chunk], valid[a:a + chunk]
        ref = np.zeros(yc.shape)
        for v in np.unique(vc[vc > 0]):
            sel = np.flatnonzero(vc == v)
            seg = xc[sel, :, :, :v].astype(np.float64)
            mu, sigma = MN.stats(seg, int(v))
            ref[sel, :, :, :v] = (seg - mu) / (sigma + MN.EPS)
        worst = max(worst, ulp_ratio(yc, ref))
    return worst
