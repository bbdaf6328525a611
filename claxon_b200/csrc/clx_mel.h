// clx_mel.h — the per-frame arithmetic of mel_kernel and mel_packed_kernel (clx_mel.cu): the real FFT of n_fft = 2N samples as a complex
// Stockham FFT of N points (radices 4, 2, 3, 5) and the even / odd split to |X[k]|^2, k <= N.  Plain C++ as well as
// CUDA, so that tools/mel_host.cpp runs the very code the kernel runs on the host (tests/test_mel_host.py).
#ifndef CLX_MEL_H
#define CLX_MEL_H
#include <stdint.h>

#ifdef __CUDACC__
#define CLX_MEL_HD __host__ __device__ __forceinline__
#else
#define CLX_MEL_HD inline
#endif

namespace clx {

struct alignas(8) MelCpx {
    float re, im;
};

CLX_MEL_HD MelCpx mel_mul(MelCpx a, MelCpx b) { return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }

// The frames of a row of n samples: 1 + n / hop reflect-padded (n > n_fft / 2, the pad torch.stft accepts), else
// 1 + (n - n_fft) / hop (n >= n_fft); 0 for a shorter row.
CLX_MEL_HD uint64_t mel_frame_count(uint64_t n, uint32_t n_fft, uint32_t hop, bool center) {
    if (center) return n > n_fft / 2 ? 1 + n / hop : 0;
    return n >= n_fft ? 1 + (n - n_fft) / hop : 0;
}

// The radix of the Stockham stage that has `left` = N / Ns points still to combine.
CLX_MEL_HD uint32_t mel_radix(uint32_t left) { return left % 4 == 0 ? 4 : left % 2 == 0 ? 2 : left % 3 == 0 ? 3 : 5; }

// v <- DFT_R(v), forward (exp(-2 pi i q r / R)), in place.
template <int R>
CLX_MEL_HD void mel_dft(MelCpx* v) {
    if (R == 2) {
        const MelCpx a = v[0], b = v[1];
        v[0] = {a.re + b.re, a.im + b.im};
        v[1] = {a.re - b.re, a.im - b.im};
    } else if (R == 4) {
        const MelCpx s02 = {v[0].re + v[2].re, v[0].im + v[2].im}, d02 = {v[0].re - v[2].re, v[0].im - v[2].im};
        const MelCpx s13 = {v[1].re + v[3].re, v[1].im + v[3].im}, d13 = {v[1].re - v[3].re, v[1].im - v[3].im};
        v[0] = {s02.re + s13.re, s02.im + s13.im};
        v[2] = {s02.re - s13.re, s02.im - s13.im};
        v[1] = {d02.re + d13.im, d02.im - d13.re};  // d02 - i d13
        v[3] = {d02.re - d13.im, d02.im + d13.re};  // d02 + i d13
    } else if (R == 3) {
        const float c = -0.5f, s = 0.866025403784438647f;  // cos, sin(2 pi / 3)
        const MelCpx p = {v[1].re + v[2].re, v[1].im + v[2].im}, m = {v[1].re - v[2].re, v[1].im - v[2].im};
        const MelCpx t = {v[0].re + c * p.re, v[0].im + c * p.im};
        v[0] = {v[0].re + p.re, v[0].im + p.im};
        v[1] = {t.re + s * m.im, t.im - s * m.re};  // t - i s m
        v[2] = {t.re - s * m.im, t.im + s * m.re};
    } else {  // R == 5
        const float c1 = 0.309016994374947424f, c2 = -0.809016994374947424f;  // cos(2 pi / 5), cos(4 pi / 5)
        const float s1 = 0.951056516295153572f, s2 = 0.587785252292473129f;   // sin(2 pi / 5), sin(4 pi / 5)
        const MelCpx p1 = {v[1].re + v[4].re, v[1].im + v[4].im}, m1 = {v[1].re - v[4].re, v[1].im - v[4].im};
        const MelCpx p2 = {v[2].re + v[3].re, v[2].im + v[3].im}, m2 = {v[2].re - v[3].re, v[2].im - v[3].im};
        const MelCpx a1 = {v[0].re + c1 * p1.re + c2 * p2.re, v[0].im + c1 * p1.im + c2 * p2.im};
        const MelCpx a2 = {v[0].re + c2 * p1.re + c1 * p2.re, v[0].im + c2 * p1.im + c1 * p2.im};
        const MelCpx b1 = {s1 * m1.re + s2 * m2.re, s1 * m1.im + s2 * m2.im};
        const MelCpx b2 = {s2 * m1.re - s1 * m2.re, s2 * m1.im - s1 * m2.im};
        v[0] = {v[0].re + p1.re + p2.re, v[0].im + p1.im + p2.im};
        v[1] = {a1.re + b1.im, a1.im - b1.re};  // a1 - i b1
        v[4] = {a1.re - b1.im, a1.im + b1.re};
        v[2] = {a2.re + b2.im, a2.im - b2.re};
        v[3] = {a2.re - b2.im, a2.im + b2.re};
    }
}

CLX_MEL_HD uint32_t mel_mulhi(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

// The Stockham stage after Ns (the product of the earlier radices) of an N-point FFT, for nf frames of N points at
// in + f N -> out + f N: butterfly j < N / R of a frame reads in[j + r N / R], twiddles them by W_{Ns R}^(r (j mod Ns)),
// takes DFT_R and writes out[(j - j mod Ns) R + j mod Ns + r Ns].  tw[i] = exp(-2 pi i i / (2N)), so W_{Ns R}^x =
// tw[2 x N / (Ns R)].  Thread `tid` of `nthreads` takes butterflies tid, tid + nthreads, ... of the nf N / R, walking
// (frame, j) without divisions; j mod Ns is taken by multiplication (exact: j and Ns are below 2^11).
template <int R>
CLX_MEL_HD void mel_pass(const MelCpx* in, MelCpx* out, const MelCpx* tw, uint32_t N, uint32_t Ns, uint32_t nf,
                         uint32_t tid, uint32_t nthreads) {
    const uint32_t m = N / R, unit = 2 * (N / (Ns * R));
    const uint32_t magic = Ns > 1 ? 0xffffffffu / Ns + 1 : 0;  // ceil(2^32 / Ns) for Ns > 1
    const uint32_t df = nthreads / m, dj = nthreads - df * m;
    uint32_t f = tid / m, j = tid - f * m;
    for (; f < nf;) {
        const uint32_t k = Ns > 1 ? j - Ns * mel_mulhi(j, magic) : 0, step = k * unit;
        const MelCpx* x = in + f * N;
        MelCpx v[R];
        v[0] = x[j];
#pragma unroll
        for (int r = 1; r < R; r++) v[r] = mel_mul(x[j + r * m], tw[r * step]);
        mel_dft<R>(v);
        MelCpx* y = out + f * N + (j - k) * R + k;
#pragma unroll
        for (int r = 0; r < R; r++) y[r * Ns] = v[r];
        j += dj;
        f += df;
        if (j >= m) {
            j -= m;
            f++;
        }
    }
}

CLX_MEL_HD void mel_stage(const MelCpx* in, MelCpx* out, const MelCpx* tw, uint32_t N, uint32_t Ns, uint32_t R,
                          uint32_t nf, uint32_t tid, uint32_t nthreads) {
    switch (R) {
        case 4: mel_pass<4>(in, out, tw, N, Ns, nf, tid, nthreads); break;
        case 2: mel_pass<2>(in, out, tw, N, Ns, nf, tid, nthreads); break;
        case 3: mel_pass<3>(in, out, tw, N, Ns, nf, tid, nthreads); break;
        default: mel_pass<5>(in, out, tw, N, Ns, nf, tid, nthreads); break;
    }
}

// |X[k]|^2, k <= N, of the real frame x of 2N samples whose N-point FFT of z[i] = x[2i] + i x[2i + 1] is Z:
// X[k] = E + W^k O, E = (Z[k] + conj Z[N - k]) / 2, O = (Z[k] - conj Z[N - k]) / 2i, W = tw[1], Z[N] = Z[0].
CLX_MEL_HD float mel_power(const MelCpx* Z, const MelCpx* tw, uint32_t N, uint32_t k) {
    const MelCpx a = Z[k == N ? 0 : k], b = Z[k == 0 ? 0 : N - k];
    const MelCpx e = {0.5f * (a.re + b.re), 0.5f * (a.im - b.im)};
    const MelCpx o = {0.5f * (a.im + b.im), 0.5f * (b.re - a.re)};
    const MelCpx x = mel_mul(tw[k], o);
    const float re = e.re + x.re, im = e.im + x.im;
    return re * re + im * im;
}

}  // namespace clx
#endif
