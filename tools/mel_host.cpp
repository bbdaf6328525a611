// mel_host.cpp — host harness for the per-frame arithmetic of mel_kernel (claxon_b200/csrc/clx_mel.h).  Test
// infrastructure only (tests/test_mel_host.py): it runs the code the kernel runs per frame, stage after stage with
// every butterfly of a stage before the next as the kernel's barriers order them, with the kernel's twiddle table.
// Build: g++ -O2 -shared -fPIC.
#include <stdint.h>

#include <cmath>
#include <utility>
#include <vector>

#include "../claxon_b200/csrc/clx_mel.h"

// The kernel's twiddle table (clx_mel.cu): exp(-2 pi i i / n_fft) in float64, stored as f32.
static void mel_twiddles(uint32_t n_fft, clx::MelCpx* tw) {
    for (uint32_t i = 0; i < n_fft; i++) {
        const double a = -2.0 * M_PI * (double)i / (double)n_fft;
        tw[i] = {(float)std::cos(a), (float)std::sin(a)};
    }
}

// |X[k]|^2 for k <= n_fft / 2 of each of n frames of n_fft samples: out[f * (n_fft / 2 + 1) + k].  The frames go
// through the stages together, as a CTA's tile does, each stage's butterflies split over `threads` threads.
extern "C" void mel_host_power(const float* x, uint32_t n, uint32_t n_fft, uint32_t threads, float* out) {
    const uint32_t N = n_fft / 2;
    std::vector<clx::MelCpx> tw(n_fft), a((size_t)n * N), b((size_t)n * N);
    mel_twiddles(n_fft, tw.data());
    for (uint64_t i = 0; i < (uint64_t)n * N; i++) a[i] = {x[2 * i], x[2 * i + 1]};
    clx::MelCpx *p = a.data(), *s = b.data();
    for (uint32_t Ns = 1, R; Ns < N; Ns *= R) {
        R = clx::mel_radix(N / Ns);
        for (uint32_t t = 0; t < threads; t++) clx::mel_stage(p, s, tw.data(), N, Ns, R, n, t, threads);
        std::swap(p, s);
    }
    for (uint32_t f = 0; f < n; f++)
        for (uint32_t k = 0; k <= N; k++) out[(uint64_t)f * (N + 1) + k] = clx::mel_power(p + (uint64_t)f * N, tw.data(), N, k);
}
