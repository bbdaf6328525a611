"""The resampled crop batch's filter (tests/spec_resample.py) and its host-side source bound (CPU only).

The float64 restatement is checked against torchaudio.functional.resample (when installed) and, loosely, against
scipy.signal.resample_poly; a crop computed from its clipped source span alone, as the device computes it, must equal the
slice of the whole file's resampled signal; clx_resample_source_bound must bound that span, checked by brute force.
"""
import numpy as np
import pytest

from claxon_b200 import _lib
from tests import spec_resample as S

PAIRS = [(44100, 16000), (48000, 16000), (8000, 16000), (22050, 24000), (96000, 44100), (16000, 22050)]


@pytest.mark.parametrize("r,R", PAIRS + [(44100, 48000), (24000, 16000), (16000, 16000)])
def test_matches_torchaudio(r, R):
    torch = pytest.importorskip("torch")
    F = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(r + R)
    for N in (1, 7, 1000, 4099):
        x = rng.standard_normal((2, N))
        y = S.resample(x, r, R)
        t = F.resample(torch.from_numpy(x), r, R).numpy()
        assert y.shape == t.shape == (2, S.out_len(N, r, R))
        assert np.abs(y - t).max(initial=0.0) < 1e-12, (r, R, N)


@pytest.mark.parametrize("r,R", PAIRS)
def test_close_to_resample_poly(r, R):
    """Away from the edges, a band-limited signal resamples to what scipy's polyphase resampler gives, within the
    difference of the two filters' passbands."""
    from scipy.signal import resample_poly
    o, n, _, _ = S.params(r, R)
    N = 40000
    tt = np.arange(N) / r
    f = 0.2 * min(r, R)  # well inside both passbands
    x = (np.sin(2 * np.pi * f * tt) + 0.5 * np.cos(2 * np.pi * 0.05 * min(r, R) * tt))[None, :]
    y = S.resample(x, r, R)[0]
    z = resample_poly(x[0], n, o)
    m = min(y.size, z.size)
    edge = 200 * max(1, n // o) + 200
    assert np.abs(y[edge:m - edge] - z[edge:m - edge]).max() < 2e-3, (r, R)


def test_taps_support():
    """Taps with |t| < 6 per phase: 34 for 44.1k -> 16k, 37 for 48k -> 16k, 13 for 8k -> 16k."""
    for (r, R), want in (((44100, 16000), 34), ((48000, 16000), 37), ((8000, 16000), 13)):
        o, n, base, w = S.params(r, R)
        k = np.arange(-w, w + o)[None, :]
        t = (k / o - np.arange(n)[:, None] / n) * base
        assert int((np.abs(t) < 6).sum(1).max()) == want
        # the others are negligible
        assert np.abs(S.taps(r, R)[np.abs(t) >= 6]).max(initial=0.0) < 1e-30


@pytest.mark.parametrize("r,R", PAIRS + [(16000, 16000), (96000, 8000)])
def test_crop_from_source_span_is_a_slice(r, R):
    """For every offset over several phase cycles (and near the end), the crop computed from its clipped source span
    alone equals the slice of the whole resampled signal; lengths and zero columns too."""
    rng = np.random.default_rng(7)
    o, n, _, w = S.params(r, R)
    N = 3 * (2 * w + o) + 101
    x = rng.standard_normal((2, N))
    y = S.resample(x, r, R)
    Nt = y.shape[1]
    offs = sorted(set(range(0, min(Nt + 1, 2 * n + 5))) | set(range(max(0, Nt - n - 3), Nt + 1)))
    for L in (1, max(1, n - 1), n + 1, 57):
        for off in offs:
            want, m = S._cut(y, off, L)
            got, m2 = S.crop_from_span(x, r, R, off, L)
            assert m == m2 == max(0, min(L, Nt - off))
            assert np.allclose(got, want, rtol=0, atol=1e-12), (r, R, L, off)
            assert not got[:, m:].any()


def test_source_bound_is_the_largest_span():
    """clx_resample_source_bound against a brute-force maximum of the clipped span over every offset of a long file;
    at most one source block above it, and exactly L at equal rates."""
    lib = _lib.load()
    for r, R in PAIRS + [(16000, 16000), (96000, 8000), (8000, 96000), (44100, 22050)]:
        o, n, _, w = S.params(r, R)
        N = 20 * (2 * w + o) + 7
        Nt = S.out_len(N, r, R)
        for L in (1, 2, n - 1 if n > 1 else 3, n, n + 1, 2 * n + 3, 500):
            most = 0
            for off in range(0, Nt + 1):
                lo, hi = S.source_span(N, r, R, off, L)
                most = max(most, hi - lo)
            bound = int(lib.clx_resample_source_bound(r, R, L))
            assert bound == S.source_bound(r, R, L)
            assert most <= bound, (r, R, L, most, bound)
            if r == R:
                assert bound == L
            elif Nt > L + 2 * n:
                assert bound - most <= o, (r, R, L, most, bound)


def test_source_bound_refusals():
    lib = _lib.load()
    for args in ((0, 16000, 10), (16000, 0, 10), (16000, 8000, 0), (655351, 16000, 10), (16000, 655351, 10)):
        assert lib.clx_resample_source_bound(*args) == 0, args
    assert lib.clx_resample_source_bound(655350, 1, 10) > 0
    assert lib.clx_resample_source_bound(655349, 1, (1 << 64) - 1) == (1 << 64) - 1  # overflow
