"""Element-wise error bounds for the float32 signal kernels that run after the decode (test helper, no tests here).

    fir_ref_bound(x, r, R, offset, m)   the resampled outputs [offset, offset + m) in float64 and each one's bound
    check_fir(dev, ref, bound)          asserts |dev - ref| <= bound everywhere; returns the worst ratio
    host_coefs / host_fir               a plain float32 FIR on the library's tap layout (for the checkers' own tests)
    fft_stages(n_fft), bin_bound(...)   the per-bin bound of |X_t[k]|^2
    check_bins(dev, ref, E, n_fft)      asserts every bin within it; returns the worst ratio

Resampler (tests/spec_resample.py's filter).  Output j = blk * n + ph is sum_k h[ph, k] x[blk * o + k], which the kernel
sums in ascending k with fmaf from 0.f, with f32(h) for h.  A term whose product is 0 leaves the sum unchanged, and the
first non-zero term is exact, so with q non-zero terms the result differs from the float64 sum by the coefficients'
rounding (at most 2^-24 sum |h||x|) and q - 1 roundings of partial sums (each at most 2^-24 sum |h||x|, to first
order).  An output that sees one impulse (q = 1) is exactly f32(h) x: within 2^-24 |h x| of the reference, which for x
= 0.5 is 2^-25 |h|.  Otherwise the bound is (T + 1) 2^-24 sum |h||x|, T the phase's tap count.  The library's taps with
|t| >= 6 are exactly 0 where the float64 restatement clips t and gets about 1e-49; TINY absorbs that, and an output
with no non-zero term must be exactly 0.

Mel power.  Let u = 2^-24 and E_t = n_fft sum_j w_j^2 x_j^2 the frame's energy, so that sum over all n_fft bins of
|X_t[k]|^2 is E_t and every |X_t[k]| <= sqrt(E_t).  Each exact step of the kernel is a multiple of a unitary map: a
Stockham stage of radix R multiplies a frame's L2 norm by sqrt(R).  So an error of relative L2 size eta made at one
step reaches the spectrum with relative size eta, and the steps' errors add (to first order).  With Z the N-point
FFT (N = n_fft / 2), |Z| = sqrt(E_t / 2), and X_k = (Z_k + conj Z_{N-k}) / 2 + W^k (Z_k - conj Z_{N-k}) / 2i gives
|dX_k| <= |dZ_k| + |dZ_{N-k}| <= sqrt(2) |dZ|: an FFT error of relative size eta is at most eta sqrt(E_t) in any bin.
Per step, in units of u:
  - windowing, f32(w x): 1.
  - a stage's twiddles: the float32 table is within u of exp(-2 pi i m / n_fft) (each component rounded once from
    float64), and a complex product, FMA-contracted or not, is within 2 sqrt(2) u |a||b|: 1 + 2 sqrt(2) < 4.
  - radix 2: one rounded add per output component, 1; radix 4: two levels of adds, the first level's errors carried
    through a sqrt(2)-times-unitary second level, 2.  With the twiddles: 5 and 6.
  - radix 3: the sums p, m (1), t = v0 - p / 2 (1), s m with s = sin(2 pi / 3) rounded (2, scaled by s < 1), the
    final add (1): under 5; with the twiddles, 9.
  - radix 5: p1, p2, m1, m2 (1), a1, a2 as two FMAs on v0 with two rounded cosines (4), b1, b2 likewise with two
    rounded sines (4), the final add (1), each scaled by constants below 1 in the L2 norm of the DFT's output: under
    8; with the twiddles, 12.
  - the even / odd split and the power: (a +- b) / 2 (1), the product with tw[k] (4), the add (1), and re^2 + im^2
    (2 u |X|^2 <= 2 u |X| sqrt(E_t)): 7 against sqrt(E_t).
KAPPA = 16 bounds every step with room for the second-order terms, so |dX_k| <= delta = KAPPA u (stages + 2)
sqrt(E_t), and ||X^_k|^2 - |X_k|^2| <= 2 |X_k| delta + delta^2.  A silent frame (E_t = 0) must give exactly 0.
"""
from __future__ import annotations

import numpy as np

from tests import spec_resample as SR

U = 2.0 ** -24
TINY = 2.0 ** -120  # above every clipped float64 tap, below every tap the library keeps
KAPPA = 16.0


# --------------------------------------------------------------------------- resampler

def _windows(x: np.ndarray, o: int, w: int, K: int, blk: np.ndarray) -> np.ndarray:
    """[C, m, K]: x[blk * o - w + i], 0 outside the file."""
    N = x.shape[1]
    idx = blk[:, None] * o - w + np.arange(K)[None, :]
    ok = (idx >= 0) & (idx < N)
    return np.where(ok[None], x[:, np.clip(idx, 0, N - 1)], 0.0)


def fir_ref_bound(x, r: int, R: int, offset: int = 0, m: int | None = None, chunk: int = 1 << 22):
    """(ref [C, m], bound [C, m]) of resample(x, r, R)[:, offset : offset + m] (the rest of the file for m None)."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    Nt = SR.out_len(x.shape[1], r, R)
    m = Nt - offset if m is None else m
    ref = np.zeros((x.shape[0], m))
    bound = np.zeros((x.shape[0], m))
    if r == R:  # a copy: exact
        ref[:] = x[:, offset:offset + m]
        return ref, bound
    o, n, _, w = SR.params(r, R)
    H = SR.taps(r, R)
    K = H.shape[1]
    nz = np.abs(H) > TINY
    T = nz.sum(1)
    step = max(1, chunk // (K * x.shape[0]))
    for a in range(0, m, step):
        blk, ph = np.divmod(np.arange(offset + a, offset + min(m, a + step)), n)
        xs = _windows(x, o, w, K, blk)
        h = H[ph]
        ref[:, a:a + len(ph)] = np.einsum("cmk,mk->cm", xs, h)
        s = np.einsum("cmk,mk->cm", np.abs(xs), np.abs(h))
        q = ((xs != 0) & nz[ph][None]).sum(-1)
        bound[:, a:a + len(ph)] = np.where(q <= 1, U * (1 + 2.0 ** -20), (T[ph] + 1)[None] * U) * s + TINY
    return ref, bound


def check_fir(dev, ref, bound, what="") -> float:
    """Asserts |dev - ref| <= bound element by element (so exactly equal where the bound is 0); returns the largest
    ratio of an error to its bound."""
    dev = np.asarray(dev, dtype=np.float64)
    err = np.abs(dev - ref)
    bad = err > bound
    if bad.any():
        i = np.unravel_index(np.argmax(bad), bad.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} outputs outside the bound, first at {i}: dev {dev[i]!r} "
                             f"ref {ref[i]!r} bound {bound[i]!r}")
    return float((err / np.where(bound > 0, bound, 1.0)).max(initial=0.0))


def host_coefs(r: int, R: int) -> np.ndarray:
    """The library's table as [n, 2w + o] float32: f32(h) where |t| < 6, else 0."""
    H = SR.taps(r, R)
    return np.where(np.abs(H) > TINY, H, 0.0).astype(np.float32)


def host_fir(x, coefs: np.ndarray, r: int, R: int, offset: int = 0, m: int | None = None) -> np.ndarray:
    """A plain float32 FIR with the table `coefs` [n, 2w + o]: acc = f32(acc + f32(c x)) in ascending k from 0."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float32))
    Nt = SR.out_len(x.shape[1], r, R)
    m = Nt - offset if m is None else m
    o, n, _, w = SR.params(r, R)
    blk, ph = np.divmod(np.arange(offset, offset + m), n)
    xs = _windows(x, o, w, coefs.shape[1], blk).astype(np.float32)
    h = coefs[ph]
    acc = np.zeros((x.shape[0], m), np.float32)
    for k in range(coefs.shape[1]):
        acc = acc + h[None, :, k] * xs[:, :, k]
    return acc


# --------------------------------------------------------------------------- mel power

def radix(left: int) -> int:
    return 4 if left % 4 == 0 else 2 if left % 2 == 0 else 3 if left % 3 == 0 else 5


def fft_stages(n_fft: int) -> int:
    """The Stockham stages of the kernel's n_fft / 2-point FFT."""
    N, Ns, s = n_fft // 2, 1, 0
    while Ns < N:
        Ns *= radix(N // Ns)
        s += 1
    return s


def frames_energy(u: np.ndarray, n_fft: int) -> np.ndarray:
    """E_t of windowed frames u [..., F, n_fft]."""
    return n_fft * (np.asarray(u, dtype=np.float64) ** 2).sum(-1)


def bin_bound(ref: np.ndarray, E: np.ndarray, n_fft: int) -> np.ndarray:
    """2 |X_k| delta + delta^2 for ref = |X_k|^2 [..., K] and E [...]."""
    delta = KAPPA * U * (fft_stages(n_fft) + 2) * np.sqrt(E)[..., None]
    return 2 * np.sqrt(ref) * delta + delta * delta


def check_bins(dev, ref, E, n_fft: int, what="") -> float:
    """Asserts every bin of dev [..., K] within bin_bound of ref; returns the largest ratio of an error to its bound."""
    return check_fir(dev, ref, bin_bound(ref, E, n_fft), what or f"n_fft {n_fft}")
