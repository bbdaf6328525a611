"""Normalised log-mel features (normalize="per_feature" / "whisper"), restated in float64 numpy, and their tolerances.

per_feature(x, v): NeMo's normalize_batch(..., "per_feature") of one segment x [..., F] (a (crop or excerpt, row, mel)
over its frames) whose first v frames are valid: mu = mean, sigma = sqrt(sum (x - mu)^2 / (v - 1)) (0 for v = 1, where
NeMo's NaN becomes 0), y = (x - mu) / (sigma + 1e-5); frames from v on are 0 (a padded batch's mask), all of them when
v = 0.

whisper(x): WhisperFeatureExtractor's map of one row's log features x [..., n_mels, F'] (natural log, the last STFT
frame already dropped): l = x / ln 10, M = the row's largest l, y = (max(l, M - 8) + 4) / 4.

Tolerances, with D the largest spec_mel log bound (spec_mel.check's tol) over the segment or row: each x is within D,
so the mean within D, each x - mu within 2D and sigma within D sqrt(v / (v - 1)) <= 2D; per_feature is within 2 D (1 +
|y|) / (sigma + 1e-5), to first order.  whisper moves l and M by at most D / ln 10 each, and (.. + 4) / 4 divides by 4:
D / (4 ln 10).  Each adds the float32 rounding of y, 2^-24 |y|.
"""
from __future__ import annotations

import numpy as np

EPS = 1e-5
LN10 = float(np.log(10.0))


def stats(x, v: int):
    """(mu, sigma) of the first v frames of each segment of x [..., F], float64, keepdims."""
    seg = np.asarray(x, dtype=np.float64)[..., :v]
    mu = seg.mean(-1, keepdims=True)
    if v < 2:
        return mu, np.zeros_like(mu)
    return mu, np.sqrt(((seg - mu) ** 2).sum(-1, keepdims=True) / (v - 1))


def per_feature(x, v: int) -> np.ndarray:
    """The per-feature map of x [..., F], frames from v on 0."""
    x = np.asarray(x, dtype=np.float64)
    y = np.zeros_like(x)
    if v > 0:
        mu, sigma = stats(x, v)
        y[..., :v] = (x[..., :v] - mu) / (sigma + EPS)
    return y


def whisper(x) -> np.ndarray:
    """The Whisper map of each row of x [..., n_mels, F']."""
    l = np.asarray(x, dtype=np.float64) / LN10
    M = l.max(axis=(-2, -1), keepdims=True)
    return (np.maximum(l, M - 8.0) + 4.0) / 4.0


def log_bound(ref, delta, log_floor: float) -> np.ndarray:
    """spec_mel.check's tolerance of log features ref (float64 spec_mel.mel) given the power bound delta."""
    return delta / np.maximum(np.exp(ref), log_floor) + 2.0 ** -20 * np.maximum(1.0, np.abs(ref))


def per_feature_tol(y, D, sigma) -> np.ndarray:
    """Per-feature tolerance of y given D (the segment's largest log bound, broadcast) and its sigma."""
    return 2.0 * D * (1.0 + np.abs(y)) / (sigma + EPS) + 2.0 ** -24 * np.abs(y)


def whisper_tol(y, D) -> np.ndarray:
    """Whisper tolerance of y given D (the row's largest log bound, broadcast)."""
    return D / (4.0 * LN10) + 2.0 ** -24 * np.abs(y)


def check(dev, ref, tol) -> float:
    """Asserts |dev - ref| <= tol elementwise; returns the largest ratio of an error to its bound."""
    err = np.abs(np.asarray(dev, dtype=np.float64) - ref)
    ratio = np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0))
    worst = float(ratio.max(initial=0.0))
    assert worst <= 1.0, (worst, np.unravel_index(np.argmax(ratio), ratio.shape))
    return worst


def within_ulp(dev, ref) -> int:
    """Asserts float32 dev within one float32 ulp of float64 ref (the ulp at the larger of the two); returns how many
    elements are not the correctly rounded value."""
    dev = np.asarray(dev, dtype=np.float32)
    r32 = np.asarray(ref, dtype=np.float64).astype(np.float32)
    ulp = np.spacing(np.maximum(np.abs(dev), np.abs(r32))).astype(np.float64)
    err = np.abs(dev.astype(np.float64) - ref)
    bad = err > ulp
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist(), float((err / ulp).max()))
    return int((dev != r32).sum())
