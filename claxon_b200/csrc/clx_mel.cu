// clx_mel.cu — mel crop batches (include/claxon_b200.h, clx_batch_create_mel_crops): the mel spectrogram of every row
// of a crop batch's [n_crops * C, L] float32 output, by one kernel after the inner batch's launch sequence.
//
// mel_kernel: one CTA per (row, tile of consecutive frames).  It reads the tile's frames from the inner output (reflect
// indexing at the row's ends with CLX_MEL_CENTER), windows them and stores each as n_fft / 2 complex points in shared
// memory; runs a Stockham FFT of n_fft / 2 points per frame, ping-ponging between two buffers (clx_mel.h); writes each
// frame's power |X[k]|^2, k <= n_fft / 2, into the free buffer; then each thread sums one (mel, frame) over the mel's
// non-zero bins, threads laid along the frames so that each mel row of the tile is stored contiguously.  Every sum has
// one fixed order and no atomics: calls are bit-identical.
//
// Mel packed batches (clx_batch_create_mel_packed) run two kernels after an inner packed or resampled packed batch:
// mel_packed_plan_kernel gives each excerpt its frame count and frame start, and mel_packed_kernel computes the frames
// of one (tile of frame columns, row) per CTA with mel_kernel's per-frame arithmetic, once over the whole tile whatever
// the excerpts in it.
//
// With CLX_MEL_NORM_PER_FEATURE or CLX_MEL_NORM_WHISPER, mel_norm_kernel follows either mel kernel and normalises the
// log features in place: per (crop or excerpt, row, mel) mean and variance over the valid frames, or Whisper's clamp
// and rescale per crop row.  The mel kernels do not change; for Whisper, mel_kernel just runs with F - 1 frames.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_mel.h"
#include "clx_scan.cuh"

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

// One CTA, SCAN_THREADS excerpts at a time: F_b = mel_frame_count(n_b) of the inner batch's length n_b (0 for an
// invalid, non-fitting or empty excerpt), start_0 = 0 and start_{b+1} = start_b + round_up_4(F_b), for b < count.
__global__ void __launch_bounds__(SCAN_THREADS)
mel_packed_plan_kernel(MelPacked mp, uint32_t n_fft, uint32_t hop, bool center) {
    __shared__ PackedSums s_warp[SCAN_THREADS / 32];
    __shared__ PackedSums s_cols;
    if (threadIdx.x == 0) s_cols = PackedSums{};
    __syncthreads();
    const uint32_t used = min(*mp.count, mp.n);
    for (uint32_t base = 0; base < used; base += SCAN_THREADS) {
        const uint32_t b = base + threadIdx.x;
        const uint64_t F = b < used ? mel_frame_count((uint64_t)mp.lengths[b], n_fft, hop, center) : 0;
        const uint64_t start = cta_scan(PackedSums{(F + 3) & ~(uint64_t)3, 0, 0, 0}, s_warp, &s_cols).cols;
        if (b < used) {
            mp.starts[b] = (int64_t)start;
            mp.frames[b] = (int64_t)F;
        }
    }
}

// Frame j of an excerpt whose n samples start at column base of the inner output's rows.
struct MelSlot {
    int64_t base, n;
    uint32_t j;
};

// mel_kernel over frame columns [t0, t0 + nf) of features row `row` of the packed layout.  Each of the tile's columns
// finds its excerpt by binary search (the ends start_b + F_b never decrease, since start_{b+1} >= start_b + F_b): the
// first b whose end passes the column holds it if start_b <= the column, else the column is an alignment gap or lies
// past the last excerpt.  The tile's frames are compacted into slots 0 .. nv - 1, the one windowing, FFT and power pass
// runs over those, and each column stores its slot's mel sums, or 0 for a column without a frame.
__global__ void __launch_bounds__(MEL_THREADS)
mel_packed_kernel(MelBuffers mb, MelPacked mp) {
    extern __shared__ MelCpx s_buf[];  // two buffers of tile * N points
    __shared__ MelSlot s_slot[MEL_MAX_TILE];
    __shared__ int32_t s_col[MEL_MAX_TILE];  // column f's slot, -1 for none
    __shared__ uint32_t s_nv;
    const uint32_t N = mb.n_fft / 2, T = mb.tile;
    const uint32_t row = blockIdx.x / mb.tiles, tile = blockIdx.x - row * mb.tiles;
    const uint64_t t0 = (uint64_t)tile * T;
    const uint32_t nf = (uint32_t)min((uint64_t)T, mb.F - t0);
    if (threadIdx.x < 32) {  // T <= 32: one warp
        const uint32_t f = threadIdx.x, used = min(*mp.count, mp.n);
        const uint64_t t = t0 + f;
        bool valid = false;
        MelSlot s{0, 0, 0};
        if (f < nf) {
            uint32_t lo = 0, hi = used;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if ((uint64_t)(mp.starts[mid] + mp.frames[mid]) > t) hi = mid;
                else lo = mid + 1;
            }
            if (lo < used && (uint64_t)mp.starts[lo] <= t) {
                valid = true;
                s = MelSlot{mp.src_starts[lo], mp.lengths[lo], (uint32_t)(t - (uint64_t)mp.starts[lo])};
            }
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, valid), slot = __popc(mask & ((1u << f) - 1));
        if (valid) s_slot[slot] = s;
        if (f < T) s_col[f] = valid ? (int32_t)slot : -1;
        if (f == 0) s_nv = __popc(mask);
    }
    __syncthreads();
    const uint32_t nv = s_nv;
    const MelCpx* tw = reinterpret_cast<const MelCpx*>(mb.tw);
    MelCpx* a = s_buf;
    MelCpx* b = s_buf + T * N;
    const uint32_t K = N + 1, P = K | 1;
    float* pw = reinterpret_cast<float*>(b);
    if (nv) {
        // 1. The frames, windowed, as in mel_kernel, each reflect-padded within its own excerpt (n > N with
        //    CLX_MEL_CENTER, n >= n_fft without: every index reflects into the excerpt once, or not at all).
        const int64_t pad = (mb.flags & CLX_MEL_CENTER) ? (int64_t)N : 0;
        const float* xr = mb.src + (uint64_t)row * mb.L;
        {
            const uint32_t df = MEL_THREADS / N, dq = MEL_THREADS - df * N;
            for (uint32_t f = threadIdx.x / N, q = threadIdx.x - f * N; f < nv;) {
                const MelSlot s = s_slot[f];
                const float* x = xr + s.base;
                const int64_t p = (int64_t)s.j * mb.hop + 2 * q - pad, L = s.n;
                float v[2];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    int64_t i = p + h;
                    i = i < 0 ? -i : i >= L ? 2 * L - 2 - i : i;
                    const float w = __ldg(mb.window + 2 * q + h);
                    v[h] = w != 0.f ? w * __ldg(x + i) : 0.f;
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
        // 2. The FFT of every slot.
        for (uint32_t Ns = 1, R; Ns < N; Ns *= R) {
            R = mel_radix(N / Ns);
            __syncthreads();
            mel_stage(a, b, tw, N, Ns, R, nv, threadIdx.x, MEL_THREADS);
            MelCpx* t = a;
            a = b;
            b = t;
        }
        __syncthreads();
        // 3. The power of bins 0 .. N of slot f at pw[f * P + k].
        pw = reinterpret_cast<float*>(b);
        const uint32_t df = MEL_THREADS / K, dk = MEL_THREADS - df * K;
        for (uint32_t f = threadIdx.x / K, k = threadIdx.x - f * K; f < nv;) {
            pw[f * P + k] = mel_power(a + f * N, tw, N, k);
            k += dk;
            f += df;
            if (k >= K) {
                k -= K;
                f++;
            }
        }
        __syncthreads();
    }
    // 4. The mel sums of every column of the tile, frames fastest; 0 where a column has no frame.
    const bool log = mb.flags & CLX_MEL_LOG;
    const uint32_t shift = __ffs(T) - 1;
    for (uint32_t i = threadIdx.x; i < mb.n_mels * T; i += MEL_THREADS) {
        const uint32_t m = i >> shift, f = i & (T - 1);
        if (f >= nf) continue;
        const int32_t sl = s_col[f];
        float acc = 0.f;
        if (sl >= 0) {
            const MelBand band = mb.bands[m];
            const float* w = mb.weights + band.w;
            const float* s = pw + (uint32_t)sl * P + band.lo;
            for (uint32_t k = 0; k < band.n; k++) acc = fmaf(__ldg(w + k), s[k], acc);
            if (log) acc = acc > mb.log_floor ? logf(acc) : mb.log_of_floor;
        }
        mb.out[((uint64_t)row * mb.n_mels + m) * mb.F + t0 + f] = acc;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// mel_norm_kernel: the CLX_MEL_NORM_* maps, in place over the log features the mel kernel wrote.  Statistics and maps
// are float64, rounded once to float32; every reduction has one fixed order and no atomics, so calls are bit-identical
// and a constant segment gives exactly 0 (its partial sums k x are exact in float64, so mu = x).

constexpr uint32_t MEL_NORM_THREADS = 512;
constexpr uint32_t MEL_NORM_MAX_CTAS = 1u << 20;  // per-feature CTAs loop over the segments past that
constexpr double MEL_LOG10_E = 0.434294481903251827651;  // 1 / ln 10

// The sum of v over a warp, by xor butterflies: every lane adds the same two values at each step, so all lanes get
// the same sum.
__device__ __forceinline__ double mel_warp_sum(double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// CLX_MEL_NORM_PER_FEATURE: one warp per segment (crop or excerpt b, row c, mel m), segments numbered b-major.  Three
// walks over the segment's contiguous frames, lane t mod 32 taking frame t: the sum, the squared deviations from the
// mean, then the map in place (a crop's frames past v written 0).  The last two walks read what the first brought
// into L1 / L2.
__device__ __forceinline__ void mel_norm_per_feature(const MelNorm& mn) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t segs = mn.n * mn.C * mn.n_mels, warps = gridDim.x * (MEL_NORM_THREADS / 32);  // (< 2^31: create)
    const uint32_t used = mn.count ? min(*mn.count, mn.n) : mn.n;
    for (uint32_t s = (blockIdx.x * MEL_NORM_THREADS + threadIdx.x) / 32; s < segs; s += warps) {
        const uint32_t rc = s / mn.n_mels;  // b C + c
        const uint32_t m = s - rc * mn.n_mels, b = rc / mn.C, c = rc - b * mn.C;
        if (b >= used) break;  // (s only grows)
        float* x;
        uint64_t v, F;
        if (mn.count) {  // packed: F_b frames at start_b, nothing else to write
            v = F = (uint64_t)mn.frames[b];
            x = mn.out + ((uint64_t)c * mn.n_mels + m) * mn.F + mn.starts[b];
        } else {  // crops: torch.stft's frame count of the crop's n_b samples, 0 for none
            const int64_t n = mn.lengths[b];
            v = n > 0 ? min(mn.F, 1 + (uint64_t)n / mn.hop) : 0;
            F = mn.F;
            x = mn.out + (uint64_t)s * mn.F;
        }
        double sum = 0.0;
        for (uint64_t t = lane; t < v; t += 32) sum += (double)x[t];
        const double mu = mel_warp_sum(sum) / (double)v;
        double dev = 0.0;
        for (uint64_t t = lane; t < v; t += 32) {
            const double d = (double)x[t] - mu;
            dev = fma(d, d, dev);
        }
        const double sigma = v > 1 ? sqrt(mel_warp_sum(dev) / (double)(v - 1)) : 0.0, den = sigma + 1e-5;
        for (uint64_t t = lane; t < F; t += 32) x[t] = t < v ? (float)(((double)x[t] - mu) / den) : 0.f;
    }
}

// CLX_MEL_NORM_WHISPER: one CTA per row of [n_mels, F'] features.  The row's largest x (the largest l as well: the
// scaling keeps the order), then y = (max(l, M - 8) + 4) / 4 in place, l = x log10(e) (within an ulp of x / ln 10 in
// float64, far below the float32 rounding).
__device__ __forceinline__ void mel_norm_whisper(const MelNorm& mn) {
    __shared__ float s_max[MEL_NORM_THREADS / 32];
    const uint64_t n = (uint64_t)mn.n_mels * mn.F;
    float* x = mn.out + (uint64_t)blockIdx.x * n;
    float hi = -INFINITY;
#pragma unroll 4
    for (uint64_t i = threadIdx.x; i < n; i += MEL_NORM_THREADS) hi = fmaxf(hi, x[i]);
    for (int o = 16; o; o >>= 1) hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x / 32] = hi;
    __syncthreads();
    hi = s_max[0];
    for (uint32_t w = 1; w < MEL_NORM_THREADS / 32; w++) hi = fmaxf(hi, s_max[w]);
    const double lo = (double)hi * MEL_LOG10_E - 8.0;
#pragma unroll 4
    for (uint64_t i = threadIdx.x; i < n; i += MEL_NORM_THREADS)
        x[i] = (float)((fmax((double)x[i] * MEL_LOG10_E, lo) + 4.0) * 0.25);
}

__global__ void __launch_bounds__(MEL_NORM_THREADS)
mel_norm_kernel(MelNorm mn) {
    if (mn.flags & CLX_MEL_NORM_WHISPER) mel_norm_whisper(mn);
    else mel_norm_per_feature(mn);
}

namespace {
cudaError_t launch_mel_norm(const MelNorm& mn, cudaStream_t stream, uint64_t* launches) {
    if (!mn.flags) return cudaSuccess;
    const uint64_t warps = MEL_NORM_THREADS / 32, segs = (uint64_t)mn.n * mn.C * mn.n_mels;
    const uint32_t ctas = (mn.flags & CLX_MEL_NORM_WHISPER)
                              ? mn.n * mn.C  // (rows < 2^31: the mel crop create's check)
                              : (uint32_t)std::min<uint64_t>(MEL_NORM_MAX_CTAS, (segs + warps - 1) / warps);
    mel_norm_kernel<<<std::max(ctas, 1u), MEL_NORM_THREADS, 0, stream>>>(mn);
    (*launches)++;
    return cudaGetLastError();
}
}  // namespace

cudaError_t mel_init() {  // the most any batch uses, so that no batch lowers another's limit
    cudaError_t e = cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MEL_SMEM);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(mel_packed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MEL_SMEM);
    return e;
}

cudaError_t launch_mel(const MelBuffers& mb, const MelNorm& mn, size_t smem, cudaStream_t stream, uint64_t* launches) {
    mel_kernel<<<mb.rows * mb.tiles, MEL_THREADS, smem, stream>>>(mb);
    (*launches)++;
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? launch_mel_norm(mn, stream, launches) : e;
}

cudaError_t launch_mel_packed(const MelBuffers& mb, const MelPacked& mp, const MelNorm& mn, size_t smem,
                              cudaStream_t stream, uint64_t* launches) {
    mel_packed_plan_kernel<<<1, SCAN_THREADS, 0, stream>>>(mp, mb.n_fft, mb.hop, (mb.flags & CLX_MEL_CENTER) != 0);
    (*launches)++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    mel_packed_kernel<<<mb.rows * mb.tiles, MEL_THREADS, smem, stream>>>(mb, mp);
    (*launches)++;
    e = cudaGetLastError();
    return e == cudaSuccess ? launch_mel_norm(mn, stream, launches) : e;
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

bool mel_params_ok(const clx_mel_params* p) {
    if (!p) return false;
    const uint32_t n_fft = p->n_fft;
    const uint32_t norm = p->flags & (CLX_MEL_NORM_PER_FEATURE | CLX_MEL_NORM_WHISPER);
    if (n_fft % 2 || n_fft < 8 || n_fft > 4096 || !smooth(n_fft / 2) || p->win_length < 1 || p->win_length > n_fft ||
        p->hop_length < 1 || p->n_mels < 1 || p->n_mels > 512 || (p->flags & ~(CLX_MEL_CENTER | CLX_MEL_LOG | norm)))
        return false;
    // a normalisation needs the log of centred frames, and takes one map
    if (norm && (norm == (CLX_MEL_NORM_PER_FEATURE | CLX_MEL_NORM_WHISPER) ||
                 (p->flags & (CLX_MEL_LOG | CLX_MEL_CENTER)) != (CLX_MEL_LOG | CLX_MEL_CENTER)))
        return false;
    return (p->flags & CLX_MEL_LOG) ? std::isfinite(p->log_floor) && p->log_floor > 0.f : p->log_floor == 0.f;
}

bool mel_tables(const clx_mel_params* p, const float* window, const float* fbank, MelTables* t) {
    if (!mel_params_ok(p) || !window || !fbank) return false;
    const uint32_t n_fft = p->n_fft, N = n_fft / 2;
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

// The frame columns of the excerpts that fit in a packed batch of B excerpts and T sample columns (DESIGN §3.6).  The
// excerpts with frames have n_b >= m, m the shortest row with a frame (n_fft / 2 + 1 with CLX_MEL_CENTER, n_fft
// without); all but the last of them take round_up_4(n_b) >= round_up_4(m) columns before the last one's start, and
// that one ends by T: k <= min(B, (T - m) / round_up_4(m) + 1) of them, and the n_b add up to T at most.  Each takes
// round_up_4(F_b) <= F_b + 3 <= n_b / hop + 4 frame columns, and the floors of n_b / hop add up to floor(T / hop) at
// most: round_up_4(floor(T / hop) + 4k) in all.
size_t mel_packed_frames(const clx_mel_params* p, size_t max_excerpts, size_t max_samples) {
    const uint64_t m = (p->flags & CLX_MEL_CENTER) ? p->n_fft / 2 + 1 : p->n_fft, m4 = (m + 3) & ~(uint64_t)3;
    if (max_samples < m) return 0;
    const uint64_t k = std::min<uint64_t>(max_excerpts, (max_samples - m) / m4 + 1);
    const unsigned __int128 cols = (unsigned __int128)(max_samples / p->hop_length) + 4 * (unsigned __int128)k + 3;
    return cols > SIZE_MAX ? SIZE_MAX : (size_t)(cols & ~(unsigned __int128)3);
}

}  // namespace clx

extern "C" size_t clx_mel_packed_frames_bound(const clx_mel_params* params, size_t max_excerpts, size_t max_samples) {
    if (!clx::mel_params_ok(params) || (params->flags & CLX_MEL_NORM_WHISPER) || max_excerpts == 0 || max_samples == 0)
        return 0;
    return clx::mel_packed_frames(params, max_excerpts, max_samples);
}
