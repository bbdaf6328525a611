"""The resampled packed batch's inner column count, clx_resample_packed_source_bound (CPU only).

The bound must cover sum_b round_up_4(span_b) over every set of excerpts that fits in T target columns.  The brute force
takes, for each excerpt length m, the largest round_up_4 of its clipped source span (tests/spec_resample.py) over the
corpus's rates and over every offset of a long file, then a DP over every split of at most T target samples into at most
B excerpts.  Splits by sum m <= T include every layout that fits, so the DP's maximum is at least the true one.
"""
import math

import numpy as np
import pytest

from claxon_b200 import _lib
from tests import spec_resample as S

RATES = [8000, 22050, 24000, 44100, 48000, 96000, 16000]


def bound(lib, rates, R, B, T):
    arr = np.array(rates or [0], dtype=np.uint32)
    return int(lib.clx_resample_packed_source_bound(arr.ctypes.data, len(rates), R, B, T))


def largest_cols(r, R, T):
    """f[m] for m in 1..T: the largest round_up_4(hi - lo) of an excerpt of m outputs of one file at rate r."""
    o, n, _, w = S.params(r, R)
    offsets = range(0, (math.ceil(w / o) + 2) * n)  # every phase, with and without the clipping at the file's start
    N = (len(offsets) + T + 2 * n) * o // n + 2 * w + 2 * o  # long enough that no excerpt reaches the end
    f = np.zeros(T + 1, dtype=np.int64)
    for m in range(1, T + 1):
        for off in offsets:
            lo, hi = S.source_span(N, r, R, off, m)
            f[m] = max(f[m], (hi - lo + 3) & ~3)
    return f


def dp_max(f, B, T):
    """max sum_b f[m_b] over at most B excerpts with m_b >= 1 and sum m_b <= T."""
    best = np.zeros(T + 1, dtype=np.int64)  # best[t]: at most k excerpts, sum <= t
    for _ in range(min(B, T)):
        nxt = best.copy()
        for t in range(1, T + 1):
            nxt[t] = max(nxt[t], max(best[t - m] + f[m] for m in range(1, t + 1)))
        best = nxt
    return int(best[T])


@pytest.mark.parametrize("R", [16000, 44100, 48000])
def test_bound_covers_brute_force(R):
    lib = _lib.load()
    rates = RATES + ([R] if R not in RATES else [])
    T_most = 48
    f = {r: largest_cols(r, R, T_most) for r in set(rates)}
    for T in (1, 2, 3, 5, 17, T_most):
        for B in (1, 2, 3, 7, 1000):
            for sub in (rates, [R], [r for r in rates if r != R][:2]):
                fm = np.max([f[r][:T + 1] for r in sub], axis=0)
                most = dp_max(fm, B, T)
                got = bound(lib, sub, R, B, T)
                assert got % 4 == 0 and got >= most, (R, sub, B, T, most, got)
                # the closed form: ceil(T * max r / R) + min(B, T) * max c_r, rounded up to 4
                k, per, c = min(B, T), 0, 0
                for r in sub:
                    o, n, _, w = S.params(r, R)
                    per = max(per, T if r == R else -(-T * o // n))
                    c = max(c, 3 if r == R else 2 * o + 2 * w + 3)
                assert got == (per + k * c + 3) & ~3, (R, sub, B, T)


def test_bound_at_one_rate_is_tight_enough():
    """All files at R: every excerpt is copied, so T plus 3 columns of alignment per excerpt."""
    lib = _lib.load()
    for B, T in ((1, 1), (4, 10), (100, 7), (3, 1 << 20)):
        assert bound(lib, [16000] * 3, 16000, B, T) == (T + 3 * min(B, T) + 3) & ~3


def test_bound_refusals_and_overflow():
    lib = _lib.load()
    good = [44100, 48000, 16000]
    for rates, R, B, T in ((good, 0, 4, 100), (good, 655351, 4, 100), (good, 16000, 0, 100), (good, 16000, 4, 0),
                           ([44100, 0, 16000], 16000, 4, 100), ([44100, 655351], 16000, 4, 100)):
        assert bound(lib, rates, R, B, T) == 0, (rates, R, B, T)
    assert lib.clx_resample_packed_source_bound(None, 3, 16000, 4, 100) == 0
    assert lib.clx_resample_packed_source_bound(None, 0, 16000, 4, 100) == (100 + 12 + 3) & ~3  # no files: as at R
    assert bound(lib, [655350, 1], 655350, 2, 3) > 0  # the limits themselves
    assert bound(lib, [96000], 8000, 4, 1 << 62) == (1 << 64) - 1  # 12 x T overflows
    assert bound(lib, [655350], 1, 1, (1 << 64) - 1) == (1 << 64) - 1


def test_symbols_exported():
    lib = _lib.load()
    for name in ("clx_batch_create_resampled_packed", "clx_resample_packed_source_bound"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS, name
