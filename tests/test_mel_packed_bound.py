"""The mel packed batch's frame columns, clx_mel_packed_frames_bound (CPU only).

The bound must cover sum_b round_up_4(F_b) over every set of excerpts that fits in T sample columns of at most B
excerpts: excerpt b fits when start_b + n_b <= T, with start_b the sum of round_up_4(n) of the excerpts before it.  The
brute force is a DP over every such split.  Excerpts without frames only move the later ones right, so it takes those
with frames alone: all but the last cost round_up_4(n) columns, the last one n.
"""
import ctypes as C

import pytest

from claxon_b200 import _lib

SIZE_MAX = (1 << 64) - 1
CENTER = 1


def r4(n):
    return (n + 3) & ~3


def frames(n, n_fft, hop, center):
    if center:
        return 1 + n // hop if n > n_fft // 2 else 0
    return 1 + (n - n_fft) // hop if n >= n_fft else 0


def params(n_fft=400, hop=160, center=True, win=None, n_mels=1, flags=None, log_floor=0.0):
    return _lib.MelParams(n_fft, n_fft if win is None else win, hop, n_mels,
                          (CENTER if center else 0) if flags is None else flags, log_floor)


def bound(lib, p, B, T):
    return int(lib.clx_mel_packed_frames_bound(C.byref(p) if p is not None else None, B, T))


def dp_max(n_fft, hop, center, B, T):
    """max sum_b round_up_4(F_b) over at most B excerpts that fit in T columns."""
    val = [r4(frames(n, n_fft, hop, center)) for n in range(T + 1)]
    # best[c]: at most k excerpts of round_up_4(n) columns each, sum <= c (the value of n grows with n, so the best n of
    # a column cost 4q is 4q itself)
    best = [0] * (T + 1)
    answer = max([val[n] for n in range(1, T + 1)] or [0])  # one excerpt
    for _ in range(B - 1):
        nxt = list(best)
        for c in range(4, T + 1):
            nxt[c] = max(nxt[c], max(best[c - q] + val[q] for q in range(4, c + 1, 4)))
        best = nxt
        answer = max([answer] + [best[T - n] + val[n] for n in range(1, T + 1)])
    return answer


@pytest.mark.parametrize("n_fft", [8, 12, 20])
@pytest.mark.parametrize("center", [True, False])
def test_bound_covers_brute_force(n_fft, center):
    lib = _lib.load()
    for hop in sorted({1, 3, n_fft - 1, n_fft, n_fft + 5}):
        for B in (1, 2, 3, 6):
            for T in (1, 2, 3, 4, 5, 7, n_fft // 2, n_fft // 2 + 1, n_fft - 1, n_fft, n_fft + 1, 2 * n_fft + 3, 41, 64):
                most = dp_max(n_fft, hop, center, B, T)
                got = bound(lib, params(n_fft, hop, center), B, T)
                assert got % 4 == 0 and got >= most, (n_fft, hop, center, B, T, most, got)
                # the closed form
                m = n_fft // 2 + 1 if center else n_fft
                k = 0 if T < m else min(B, (T - m) // r4(m) + 1)
                assert got == (0 if k == 0 else r4(T // hop + 4 * k)), (n_fft, hop, center, B, T)


def test_bound_at_the_workload():
    """4.8 M columns at 16 kHz, 25 excerpts, hop 160: 30 000 frames and 4 columns of slack per excerpt."""
    lib = _lib.load()
    assert bound(lib, params(400, 160, True), 25, 4_800_000) == r4(30_000 + 100)
    assert bound(lib, params(400, 160, False), 25, 4_800_000) == r4(30_000 + 100)
    assert bound(lib, params(400, 160, True), 1 << 29, 4_800_000) == r4(30_000 + 4 * (4_799_799 // 204 + 1))


def test_bound_refusals_and_overflow():
    lib = _lib.load()
    assert bound(lib, None, 4, 100) == 0
    for kw in (dict(n_fft=402), dict(n_fft=401), dict(n_fft=6, win=6), dict(n_fft=8192, win=400), dict(n_fft=28, win=20),
               dict(win=0), dict(win=401), dict(hop=0), dict(n_mels=0), dict(n_mels=513), dict(flags=4),
               dict(flags=3, log_floor=0.0), dict(flags=3, log_floor=float("nan")), dict(log_floor=1e-10)):
        assert bound(lib, params(**kw), 4, 100) == 0, kw
    assert bound(lib, params(), 0, 100) == 0 and bound(lib, params(), 4, 0) == 0
    assert bound(lib, params(), 4, 200) == 0  # no frame: 200 <= n_fft / 2
    assert bound(lib, params(), 4, 201) == 8  # r4(201 // 160 + 4)
    assert bound(lib, params(center=False), 4, 399) == 0 and bound(lib, params(center=False), 4, 400) == 8
    assert bound(lib, params(flags=3, log_floor=1e-10), 4, 201) == 8  # r4(201 // 160 + 4)
    assert bound(lib, params(8, 1), SIZE_MAX, SIZE_MAX) == SIZE_MAX
    assert bound(lib, params(8, 1), 1, SIZE_MAX - 8) == SIZE_MAX - 3  # r4(T + 4) still fits


def test_symbols_exported():
    lib = _lib.load()
    for name in ("clx_batch_create_mel_packed", "clx_mel_packed_frames_bound", "clx_batch_mel_frames"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS, name
