"""The resampled crop batch's filter and crop semantics, restated in float64 numpy (no torchaudio needed).

resample(x, r, R) is torchaudio.functional.resample(x, r, R) with its defaults (lowpass_filter_width 6, rolloff 0.99,
sinc_interp_hann): with g = gcd(r, R), o = r / g and n = R / g, output j = blk * n + ph is
sum_k h[ph, k] * x[blk * o + k] over k in [-w, w + o), samples outside [0, N) reading 0, and there are
ceil(N * n / o) outputs.  A crop at rate R is a slice of the whole file's resampled signal.
"""
from __future__ import annotations

import functools
import math

import numpy as np

WIDTH = 6        # lowpass_filter_width
ROLLOFF = 0.99


def params(r: int, R: int):
    """(o, n, base, w) of the rate pair r -> R."""
    g = math.gcd(r, R)
    o, n = r // g, R // g
    base = min(o, n) * ROLLOFF
    return o, n, base, math.ceil(WIDTH * o / base)


@functools.lru_cache(maxsize=None)
def taps(r: int, R: int) -> np.ndarray:
    """h[ph, k + w] for ph in [0, n), k in [-w, w + o) (read-only)."""
    o, n, base, w = params(r, R)
    k = np.arange(-w, w + o, dtype=np.float64)[None, :]
    ph = np.arange(n, dtype=np.float64)[:, None]
    t = np.clip((k / o - ph / n) * base, -WIDTH, WIDTH)
    pt = t * np.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        sinc = np.where(t == 0, 1.0, np.sin(pt) / pt)
    h = sinc * np.cos(t * np.pi / (2 * WIDTH)) ** 2 * base / o
    h.flags.writeable = False
    return h


def out_len(N: int, r: int, R: int) -> int:
    if r == R:
        return N
    o, n, _, _ = params(r, R)
    return -(-N * n // o)


def resample(x: np.ndarray, r: int, R: int) -> np.ndarray:
    """[C, N] -> [C, ceil(N * n / o)], float64."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    if r == R:
        return x.copy()
    o, n, _, w = params(r, R)
    C_, N = x.shape
    Nt = out_len(N, r, R)
    blocks = -(-Nt // n)
    K = 2 * w + o
    pad = np.zeros((C_, blocks * o + K), dtype=np.float64)
    pad[:, w:w + N] = x  # pad[i] = x[i - w]
    win = np.lib.stride_tricks.sliding_window_view(pad, K, axis=1)[:, ::o][:, :blocks]  # [C, blocks, K]
    y = np.einsum("cbk,pk->cbp", win, taps(r, R)).reshape(C_, blocks * n)
    return y[:, :Nt]


def source_span(N: int, r: int, R: int, offset: int, L: int):
    """[lo, hi): the samples of x that outputs [offset, offset + min(L, N_t - offset)) read, clipped to [0, N) (an
    empty span at N for an empty crop)."""
    Nt = out_len(N, r, R)
    m = min(L, Nt - offset)
    if m <= 0:
        return N, N
    if r == R:
        return offset, offset + m
    o, n, _, w = params(r, R)
    b0, b1 = offset // n, (offset + m - 1) // n
    return max(0, b0 * o - w), min(N, b1 * o + w + o)


def source_bound(r: int, R: int, L: int) -> int:
    """The longest source span of a crop of L outputs: L when r == R, else (floor((L - 1) / n) + 2) * o + 2w."""
    if r == R:
        return L
    o, n, _, w = params(r, R)
    return ((L - 1) // n + 2) * o + 2 * w


def crop(x: np.ndarray, r: int, R: int, offset: int, L: int):
    """(out [C, L], length): resample(x, r, R)[:, offset : offset + L], zero past the end."""
    y = resample(x, r, R)
    return _cut(y, offset, L)


def _cut(y: np.ndarray, offset: int, L: int):
    m = max(0, min(L, y.shape[1] - offset))
    out = np.zeros((y.shape[0], L), dtype=np.float64)
    out[:, :m] = y[:, offset:offset + m]
    return out, m


def crop_from_span(x: np.ndarray, r: int, R: int, offset: int, L: int):
    """The same crop computed from the clipped source span alone, as the device does: x[lo:hi] with every sample
    outside it reading 0."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    N = x.shape[1]
    lo, hi = source_span(N, r, R, offset, L)
    m = max(0, min(L, out_len(N, r, R) - offset))
    out = np.zeros((x.shape[0], L), dtype=np.float64)
    if m == 0:
        return out, 0
    if r == R:
        out[:, :m] = x[:, lo:hi]
        return out, m
    o, n, _, w = params(r, R)
    blk, ph = np.divmod(np.arange(offset, offset + m), n)
    i = (blk * o - lo)[:, None] + np.arange(-w, w + o)[None, :]  # [m, 2w + o]: where each tap reads in the span
    ok = (i >= 0) & (i < hi - lo)
    coef = np.where(ok, taps(r, R)[ph], 0.0)
    out[:, :m] = np.einsum("cmk,mk->cm", x[:, lo:hi][:, np.where(ok, i, 0)], coef)
    return out, m
