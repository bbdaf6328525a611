"""The mel crop batch's features, restated in float64 numpy (no torchaudio needed).

mel(x) is torchaudio.transforms.MelSpectrogram with power 2, normalized False, pad 0, onesided and pad_mode "reflect",
applied to x [..., L]: with center, each row is reflect-padded by n_fft / 2 on each side; frame t is samples
[t hop, t hop + n_fft) of the padded row times the window placed at (n_fft - win_length) // 2, zeros around it;
mel[m, t] = sum_k fbank[k, m] |rfft(frame t)[k]|^2; with log_floor, ln(max(mel, log_floor)).
"""
from __future__ import annotations

import numpy as np


def n_frames(L: int, n_fft: int, hop: int, center: bool) -> int:
    return 1 + L // hop if center else 1 + (L - n_fft) // hop


def frames(x, n_fft: int, hop: int, window, center: bool) -> np.ndarray:
    """The windowed frames of every row of x [..., L]: [..., F, n_fft], float64."""
    x = np.asarray(x, dtype=np.float64)
    window = np.asarray(window, dtype=np.float64)
    L = x.shape[-1]
    if center:
        if L <= n_fft // 2:
            raise ValueError("reflect padding needs more than n_fft / 2 samples")
        x = np.pad(x, [(0, 0)] * (x.ndim - 1) + [(n_fft // 2, n_fft // 2)], mode="reflect")
    elif L < n_fft:
        raise ValueError("a frame needs n_fft samples")
    F = n_frames(L, n_fft, hop, center)
    w = np.zeros(n_fft)
    w0 = (n_fft - window.size) // 2
    w[w0:w0 + window.size] = window
    idx = np.arange(F)[:, None] * hop + np.arange(n_fft)[None, :]
    return x[..., idx] * w


def power(x, n_fft: int, hop: int, window, center: bool) -> np.ndarray:
    """|X_t[k]|^2: [..., F, n_fft // 2 + 1]."""
    return np.abs(np.fft.rfft(frames(x, n_fft, hop, window, center), axis=-1)) ** 2


def mel(x, n_fft: int, hop: int, window, fbank, center: bool = True, log_floor: float | None = None) -> np.ndarray:
    """The features of x [..., L]: [..., n_mels, F]."""
    m = np.swapaxes(power(x, n_fft, hop, window, center) @ np.asarray(fbank, dtype=np.float64), -1, -2)
    return m if log_floor is None else np.log(np.maximum(m, log_floor))


def bound(x, n_fft: int, hop: int, window, fbank, center: bool = True) -> np.ndarray:
    """The power output's tolerance: 2^-16 A_m E_t, with E_t = n_fft sum_j u_t[j]^2 (u_t the windowed frame), which
    bounds every bin's power, and A_m = sum_k |fbank[k, m]|: [..., n_mels, F]."""
    u = frames(x, n_fft, hop, window, center)
    E = n_fft * (u * u).sum(-1)
    A = np.abs(np.asarray(fbank, dtype=np.float64)).sum(0)
    return 2.0 ** -16 * A[:, None] * E[..., None, :]


def check(dev, ref, delta, log_floor: float | None = None) -> float:
    """Asserts dev within the tolerance of ref (delta the power bound), and for power outputs each element of at least
    1e-3 of its frame's largest mel within 1e-4 relative.  Returns the largest ratio of an error to its bound."""
    dev = np.asarray(dev, dtype=np.float64)
    err = np.abs(dev - ref)
    if log_floor is None:
        tol = delta
        big = ref >= 1e-3 * ref.max(axis=-2, keepdims=True)
        rel = np.where(big & (ref > 0), err / np.where(ref > 0, ref, 1.0), 0.0)
        assert rel.max(initial=0.0) <= 1e-4, rel.max()
    else:
        tol = delta / np.maximum(np.exp(ref), log_floor) + 2.0 ** -20 * np.maximum(1.0, np.abs(ref))
    ratio = np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0))
    worst = float(ratio.max(initial=0.0))
    assert worst <= 1.0, (worst, np.unravel_index(np.argmax(ratio), ratio.shape))
    return worst
