"""The element-wise checkers of tests/spec_signal.py, and the FLAC writer of tests/pcm_flac.py, on the CPU.

A checker is only worth its bound if it accepts what a correct float32 kernel computes and rejects what a subtly wrong
one computes.  Accepted: a plain float32 FIR on the library's tap layout (impulses and full-scale noise, every rate pair
the GPU tests use), and the mel kernel's own per-frame code compiled for the host (tools/mel_host.cpp) at every n_fft
the batches accept.  Rejected: the mutations the loose bounds of the older tests let through (single taps dropped,
moved or swapped between phases; bins 0 and N zeroed; a quiet bin off by a small relative amount).
"""
import hashlib

import numpy as np
import pytest

import claxon_b200 as cb
from oracle import oracle as O
from tests import pcm_flac as P
from tests import spec_decode as SD
from tests import spec_resample as SR
from tests import spec_signal as S
from tests.test_mel_host import harness, supported  # noqa: F401  (the host build of clx_mel.h)

PAIRS = [(48000, 16000), (44100, 16000), (22050, 16000), (16000, 48000), (8000, 44100), (96000, 1000), (96000, 50)]


# --------------------------------------------------------------------------- A. FLAC files from given PCM

def _pcm(C_, N, bps, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(-(1 << (bps - 1)), 1 << (bps - 1), (C_, N))
    x[:, N // 3:N // 2] = 0                               # silent blocks: constant subframes
    x[0, :3] = [-(1 << (bps - 1)), (1 << (bps - 1)) - 1, 0]  # both extremes
    return x


@pytest.mark.parametrize("bps,C_,rate,bs,N", [(8, 1, 1, 16, 100), (12, 2, 44100, 1024, 5000), (16, 4, 96000, 576, 3001),
                                              (20, 2, 655350, 4608, 4608), (24, 1, 12345, 192, 1000),
                                              (16, 8, 16000, 4096, 20000)])
def test_pcm_flac_round_trip(bps, C_, rate, bs, N):
    """cb.index accepts the file; the oracle and spec_decode decode it back exactly; the MD5 is that of the PCM."""
    pcm = _pcm(C_, N, bps, bps * 7 + C_)
    data = P.flac_from_pcm(pcm, bps, rate, bs)
    nb = (bps + 7) // 8
    md5 = hashlib.md5(b"".join(int(v).to_bytes(4, "little", signed=True)[:nb] for v in pcm.T.reshape(-1))).digest()
    idx = cb.index(data)
    f = idx[0]
    assert (f.length, f.info.sample_rate, f.info.channels, f.info.bits_per_sample) == (N, rate, C_, bps)
    assert bytes(f.info.md5sum) == md5
    st, si, first = O.open_stream(data)
    assert st == 0 and si.samples == N and bytes(si.md5sum) == md5
    st, nf, out = O.decode_stream(data, first, N * C_ + 16)
    assert st == 0 and nf == -(-N // bs)
    got = np.concatenate([out[C_ * a:C_ * min(N, a + bs)].reshape(C_, -1) for a in range(0, N, bs)], axis=1)
    assert np.array_equal(got, pcm)
    pos, blocks = first, []
    for _ in range(nf):
        kind, (ch, n) = SD.decode_frame(data[pos:].tobytes())
        assert kind == "ok"
        blocks.append(np.array(ch))
        pos += n
    assert pos == data.size and np.array_equal(np.concatenate(blocks, axis=1), pcm)


def test_pcm_flac_refusals():
    for args in ((np.zeros((1, 10)), 16, 0), (np.zeros((1, 10)), 16, 655351), (np.zeros((9, 10)), 16, 8000),
                 (np.full((1, 10), 128), 8, 8000), (np.zeros((1, 10)), 32, 8000)):
        with pytest.raises(ValueError):
            P.flac_from_pcm(*args)


# --------------------------------------------------------------------------- B. the resampler's bound

def impulses(N, r, R, C_=1, seed=0):
    """Impulses of 0.5 spaced more than 2w + o apart, at a spread of residues mod o (every one when o is small)."""
    o, _, _, w = SR.params(r, R)
    S_ = 2 * w + o + 1
    S_ += (1 - S_) % o if o > 1 else 0  # S = 1 mod o: consecutive impulses step through the residues
    x = np.zeros((C_, N))
    for c in range(C_):
        x[c, c * 7 + S_:N - S_:S_] = 0.5
    return x


def test_fir_bound_accepts_a_float32_fir():
    worst = {"impulse": 0.0, "noise": 0.0}
    rng = np.random.default_rng(5)
    for r, R in PAIRS:
        o, n, _, w = SR.params(r, R)
        coefs = S.host_coefs(r, R)
        N = min(40 * (2 * w + o), 200000)
        x = impulses(N, r, R, 2)
        m = min(SR.out_len(N, r, R), 3000)
        ref, bound = S.fir_ref_bound(x, r, R, 0, m)
        worst["impulse"] = max(worst["impulse"], S.check_fir(S.host_fir(x, coefs, r, R, 0, m), ref, bound, (r, R)))
        assert (ref != 0).any()
        noise = rng.integers(-32768, 32768, (1, min(N, 8 * (2 * w + o)))) / 32768.0
        ref, bound = S.fir_ref_bound(noise, r, R, 0, min(200, SR.out_len(noise.shape[1], r, R)))
        dev = S.host_fir(noise, coefs, r, R, 0, ref.shape[1])
        worst["noise"] = max(worst["noise"], S.check_fir(dev, ref, bound, (r, R)))
    print(f"float32 FIR, worst error / bound: {worst}")  # an impulse's is f32(h)'s rounding: up to 1


def _impulse_case(r, R):
    o, n, _, w = SR.params(r, R)
    x = impulses(60 * (2 * w + o), r, R)
    ref, bound = S.fir_ref_bound(x, r, R)
    return x, ref, bound


@pytest.mark.parametrize("mutation", ["outer-taps", "shifted-tap", "swapped-phases"])
def test_fir_bound_rejects_wrong_taps(mutation):
    r, R = (48000, 16000) if mutation != "swapped-phases" else (44100, 16000)
    x, ref, bound = _impulse_case(r, R)
    coefs = S.host_coefs(r, R)
    S.check_fir(S.host_fir(x, coefs, r, R), ref, bound)
    bad = coefs.copy()
    if mutation == "outer-taps":  # the outermost non-zero tap on each side of every phase
        for ph in range(bad.shape[0]):
            k = np.flatnonzero(bad[ph])
            bad[ph, [k[0], k[-1]]] = 0
    elif mutation == "shifted-tap":  # one tap one place later
        k = np.flatnonzero(bad[0])[3]
        bad[0, k + 1], bad[0, k] = bad[0, k], bad[0, k + 1]
    else:
        bad[[0, 1]] = bad[[1, 0]]
    with pytest.raises(AssertionError):
        S.check_fir(S.host_fir(x, bad, r, R), ref, bound, mutation)
    if mutation == "outer-taps":  # what the older absolute tolerance of 1e-5 accepts
        assert np.abs(S.host_fir(x, bad, r, R) - ref).max() <= 1e-5


# --------------------------------------------------------------------------- C. the per-bin bound of the mel power

def host_signals(n_fft, rng):
    t = np.arange(n_fft)
    k = max(1, n_fft // 7)
    sq = np.where((t // 5) % 2, 1.0, -1.0)
    imp = np.zeros(n_fft)
    imp[[0, n_fft // 3]] = [1.0, -0.5]
    mixed = rng.uniform(-0.3, 0.3, n_fft) + 0.3 + 0.3 * (-1.0) ** t  # bins 0 and N well above the rest
    return np.stack([rng.uniform(-1, 1, n_fft), mixed, np.cos(2 * np.pi * k * t / n_fft), np.ones(n_fft),
                     (-1.0) ** t, imp, sq, np.zeros(n_fft)]).astype(np.float32)


def host_power(harness, x):
    n, n_fft = x.shape
    out = np.empty((n, n_fft // 2 + 1), np.float32)
    harness.mel_host_power(np.ascontiguousarray(x).ctypes.data, n, n_fft, 256, out.ctypes.data)
    return out


def test_bin_bound_accepts_the_host_build(harness):  # noqa: F811
    rng = np.random.default_rng(9)
    worst, at = 0.0, None
    for n_fft in supported():
        x = host_signals(n_fft, rng)
        ref = np.abs(np.fft.rfft(x.astype(np.float64), axis=1)) ** 2
        ratio = S.check_bins(host_power(harness, x), ref, S.frames_energy(x, n_fft), n_fft)
        if ratio > worst:
            worst, at = ratio, n_fft
    print(f"mel host build, worst error / bound: {worst:.3g} (n_fft {at})")
    assert worst < 0.5


def _quiet_bin_case(n_fft, level):
    """One frame: a tone on bin N / 2 and one on bin N / 3 with |X|^2 = level E_t."""
    t = np.arange(n_fft)
    a = np.sqrt(2 * level / (1 - 2 * level))  # |X_k|^2 / E_t = a^2 / (2 (1 + a^2))
    x = (np.cos(2 * np.pi * (n_fft // 4) * t / n_fft) + a * np.cos(2 * np.pi * (n_fft // 6) * t / n_fft))
    return x[None].astype(np.float32), n_fft // 6


@pytest.mark.parametrize("mutation", ["bin-0", "bin-N", "1e-2-times-1.001", "1e-6-doubled"])
def test_bin_bound_rejects_wrong_bins(harness, mutation):  # noqa: F811
    for n_fft in (8, 30, 400, 480, 3750, 4096):
        if mutation.startswith("bin"):
            x = host_signals(n_fft, np.random.default_rng(1))[1:2]
            k, level = (0 if mutation == "bin-0" else n_fft // 2), None
        else:
            level = 1e-2 if mutation.startswith("1e-2") else 1e-6
            x, k = _quiet_bin_case(n_fft, level)
        ref = np.abs(np.fft.rfft(x.astype(np.float64), axis=1)) ** 2
        E = S.frames_energy(x, n_fft)
        if level is not None:
            assert abs(ref[0, k] / E[0] - level) < 0.01 * level
        dev = host_power(harness, x)
        S.check_bins(dev, ref, E, n_fft)
        bad = dev.copy()
        bad[0, k] = 0 if level is None else bad[0, k] * (1.001 if level == 1e-2 else 2)
        with pytest.raises(AssertionError):
            S.check_bins(bad, ref, E, n_fft, mutation)
        if level == 1e-6:  # what the older power tolerance, 2^-16 A E_t with A = 1, accepts
            assert abs(bad[0, k] - ref[0, k]) <= 2.0 ** -16 * E[0]
