"""CPU test of mel_kernel's per-frame arithmetic (claxon_b200/csrc/clx_mel.h).

The kernel's real FFT (a Stockham FFT of n_fft / 2 complex points, radices 4, 2, 3 and 5, and the even / odd split to
the power of bins 0 .. n_fft / 2) is compiled for the host (tools/mel_host.cpp, with the kernel's float64-built twiddle
table) and checked against numpy.fft.rfft in float64 for every n_fft the batch accepts, within the power tolerance of
tests/spec_mel.py: 2^-16 n_fft sum(x^2).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "tools", "scratch", "mel_host.so")
SRC = os.path.join(ROOT, "tools", "mel_host.cpp")
HDR = os.path.join(ROOT, "claxon_b200", "csrc", "clx_mel.h")


def supported():
    def smooth(n):
        for p in (2, 3, 5):
            while n % p == 0:
                n //= p
        return n == 1
    return [n for n in range(8, 4097, 2) if smooth(n // 2)]


@pytest.fixture(scope="module")
def harness():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", SO, SRC])
    L = C.CDLL(SO)
    L.mel_host_power.restype = None
    L.mel_host_power.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    return L


def test_every_supported_n_fft(harness):
    sizes = supported()
    assert 400 in sizes and 4096 in sizes and 30 in sizes and 402 not in sizes and len(sizes) == 107
    rng = np.random.default_rng(3)
    worst = 0.0
    for n in sizes:
        x = rng.standard_normal((4, n)).astype(np.float32)
        x[1] = 0.0                                      # zeros give exact zeros
        x[2] = np.cos(2 * np.pi * 3 * np.arange(n) / n)  # one bin
        x[3, : n // 2] = 0.0
        out = np.empty((4, n // 2 + 1), np.float32)
        harness.mel_host_power(x.ctypes.data, 4, n, 256, out.ctypes.data)  # mel_kernel's CTA of 256 threads
        x64 = x.astype(np.float64)
        ref = np.abs(np.fft.rfft(x64, axis=1)) ** 2
        E = n * (x64 ** 2).sum(1, keepdims=True)
        assert not out[1].any(), n
        bound = 2.0 ** -16 * E
        err = np.abs(out - ref)
        assert (err <= bound).all(), (n, (err / np.maximum(bound, 1e-300)).max())
        worst = max(worst, float((err[[0, 2, 3]] / bound[[0, 2, 3]]).max()))
    assert worst < 0.05, worst
