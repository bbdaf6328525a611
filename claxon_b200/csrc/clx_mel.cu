// clx_mel.cu — mel crop batches (include/claxon_b200.h, clx_batch_create_mel_crops): the mel spectrogram of every row
// of a crop batch's [n_crops * C, L] float32 output, by one kernel after the inner batch's launch sequence.
//
// mel_kernel: one CTA per (row, tile of consecutive frames).  It reads the tile's frames from the inner output (reflect
// indexing at the row's ends with CLX_MEL_CENTER), windows them and stores each as n_fft / 2 complex points in shared
// memory; runs a Stockham FFT of n_fft / 2 points per frame, ping-ponging between two buffers (clx_mel.h); writes each
// frame's power |X[k]|^2, k <= n_fft / 2, into the free buffer; then each thread sums one (mel, frame) over the mel's
// non-zero bins, threads laid along the frames so that each mel row of the tile is stored contiguously.  Every sum has
// one fixed order and no atomics: calls are bit-identical.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_mel.h"

namespace clx {

constexpr uint32_t MEL_THREADS = 256;
constexpr uint32_t MEL_MAX_TILE = 32;
constexpr size_t MEL_SMEM = 64 * 1024;  // the two FFT buffers of a tile, at most

__global__ void __launch_bounds__(MEL_THREADS)
mel_kernel(MelBuffers mb) {
    extern __shared__ MelCpx s_buf[];  // two buffers of tile * N points
    const uint32_t N = mb.n_fft / 2, T = mb.tile;
    const uint32_t row = blockIdx.x / mb.tiles, tile = blockIdx.x - row * mb.tiles;
    const uint64_t t0 = (uint64_t)tile * T;
    const uint32_t nf = (uint32_t)min((uint64_t)T, mb.F - t0);
    const float* x = mb.src + (uint64_t)row * mb.L;
    const MelCpx* tw = reinterpret_cast<const MelCpx*>(mb.tw);
    MelCpx* a = s_buf;
    MelCpx* b = s_buf + T * N;
    // 1. The frames, windowed: point q of frame f is samples 2q, 2q + 1 of it.  With CLX_MEL_CENTER the row is
    //    reflect-padded by N on each side (L > N: every index reflects into the row once).  Each loop below walks its
    //    (frame, index) pairs by steps of MEL_THREADS without dividing.
    const int64_t pad = (mb.flags & CLX_MEL_CENTER) ? (int64_t)N : 0, L = (int64_t)mb.L;
    {
        const uint32_t df = MEL_THREADS / N, dq = MEL_THREADS - df * N;
        for (uint32_t f = threadIdx.x / N, q = threadIdx.x - f * N; f < nf;) {
            const int64_t p = (int64_t)(t0 + f) * mb.hop + 2 * q - pad;
            float v[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                int64_t s = p + h;
                s = s < 0 ? -s : s >= L ? 2 * L - 2 - s : s;
                const float w = __ldg(mb.window + 2 * q + h);
                v[h] = w != 0.f ? w * __ldg(x + s) : 0.f;
            }
            a[f * N + q] = MelCpx{v[0], v[1]};
            q += dq;
            f += df;
            if (q >= N) {
                q -= N;
                f++;
            }
        }
    }
    // 2. The FFT of every frame, one stage after the other.
    for (uint32_t Ns = 1, R; Ns < N; Ns *= R) {
        R = mel_radix(N / Ns);
        __syncthreads();
        mel_stage(a, b, tw, N, Ns, R, nf, threadIdx.x, MEL_THREADS);
        MelCpx* t = a;
        a = b;
        b = t;
    }
    __syncthreads();
    // 3. The power of bins 0 .. N of frame f at pw[f * P + k], P odd so that a warp's reads of one bin across frames
    //    fall in distinct banks.
    const uint32_t K = N + 1, P = K | 1;
    float* pw = reinterpret_cast<float*>(b);
    {
        const uint32_t df = MEL_THREADS / K, dk = MEL_THREADS - df * K;
        for (uint32_t f = threadIdx.x / K, k = threadIdx.x - f * K; f < nf;) {
            pw[f * P + k] = mel_power(a + f * N, tw, N, k);
            k += dk;
            f += df;
            if (k >= K) {
                k -= K;
                f++;
            }
        }
    }
    __syncthreads();
    // 4. The mel sums, frames fastest (T is a power of two).
    const bool log = mb.flags & CLX_MEL_LOG;
    const uint32_t shift = __ffs(T) - 1;
    for (uint32_t i = threadIdx.x; i < mb.n_mels * T; i += MEL_THREADS) {
        const uint32_t m = i >> shift, f = i & (T - 1);
        if (f >= nf) continue;
        const MelBand band = mb.bands[m];
        const float* w = mb.weights + band.w;
        const float* s = pw + f * P + band.lo;
        float acc = 0.f;
        for (uint32_t k = 0; k < band.n; k++) acc = fmaf(__ldg(w + k), s[k], acc);
        if (log) acc = acc > mb.log_floor ? logf(acc) : mb.log_of_floor;
        mb.out[((uint64_t)row * mb.n_mels + m) * mb.F + t0 + f] = acc;
    }
}

cudaError_t mel_init() {  // the most any batch uses, so that no batch lowers another's limit
    return cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MEL_SMEM);
}

cudaError_t launch_mel(const MelBuffers& mb, size_t smem, cudaStream_t stream, uint64_t* launches) {
    mel_kernel<<<mb.rows * mb.tiles, MEL_THREADS, smem, stream>>>(mb);
    (*launches)++;
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side: the checks and tables of clx_batch_create_mel_crops.

namespace {
bool smooth(uint32_t n) {  // no prime factor above 5
    for (uint32_t p : {2u, 3u, 5u})
        while (n % p == 0) n /= p;
    return n == 1;
}
}  // namespace

bool mel_tables(const clx_mel_params* p, const float* window, const float* fbank, size_t num_frames, MelTables* t) {
    if (!p || !window || !fbank) return false;
    const uint32_t n_fft = p->n_fft, N = n_fft / 2;
    if (n_fft % 2 || n_fft < 8 || n_fft > 4096 || !smooth(N) || p->win_length < 1 || p->win_length > n_fft ||
        p->hop_length < 1 || p->n_mels < 1 || p->n_mels > 512 || (p->flags & ~(CLX_MEL_CENTER | CLX_MEL_LOG)))
        return false;
    if ((p->flags & CLX_MEL_LOG) ? !(std::isfinite(p->log_floor) && p->log_floor > 0.f) : p->log_floor != 0.f)
        return false;
    if ((p->flags & CLX_MEL_CENTER) ? num_frames <= N : num_frames < n_fft) return false;
    t->F = (p->flags & CLX_MEL_CENTER) ? 1 + num_frames / p->hop_length : 1 + (num_frames - n_fft) / p->hop_length;
    t->window.assign(n_fft, 0.f);
    const uint32_t w0 = (n_fft - p->win_length) / 2;
    for (uint32_t i = 0; i < p->win_length; i++) {
        if (!std::isfinite(window[i])) return false;
        t->window[w0 + i] = window[i];
    }
    const size_t n_mels = p->n_mels;
    for (size_t i = 0; i < (size_t)(N + 1) * n_mels; i++)
        if (!std::isfinite(fbank[i])) return false;
    t->bands.resize(n_mels);
    t->weights.clear();
    for (size_t m = 0; m < n_mels; m++) {  // the bins [lo, hi) between the first and last non-zero weight
        uint32_t lo = N + 1, hi = 0;
        for (uint32_t k = 0; k <= N; k++)
            if (fbank[(size_t)k * n_mels + m] != 0.f) {
                lo = std::min(lo, k);
                hi = k + 1;
            }
        if (hi == 0) lo = 0;
        t->bands[m] = MelBand{lo, hi - lo, (uint32_t)t->weights.size()};
        for (uint32_t k = lo; k < hi; k++) t->weights.push_back(fbank[(size_t)k * n_mels + m]);
    }
    if (t->weights.empty()) t->weights.push_back(0.f);
    t->tw.resize(2 * (size_t)n_fft);
    for (uint32_t i = 0; i < n_fft; i++) {
        const double a = -2.0 * M_PI * (double)i / (double)n_fft;
        t->tw[2 * i] = (float)std::cos(a);
        t->tw[2 * i + 1] = (float)std::sin(a);
    }
    // The largest power of two of frames, up to MEL_MAX_TILE, whose two buffers fit in MEL_SMEM (one frame at least:
    // 2 * 2048 points of 8 bytes at n_fft 4096).
    t->tile = MEL_MAX_TILE;
    while (t->tile > 1 && 2 * (size_t)t->tile * N * sizeof(MelCpx) > MEL_SMEM) t->tile /= 2;
    t->smem = 2 * (size_t)t->tile * N * sizeof(MelCpx);
    return true;
}

}  // namespace clx
