// clx_resample.cu — resampled crop batches (include/claxon_b200.h, clx_batch_create_resampled_crops): [B, C, L] crops of
// a corpus whose files have different sample rates, all at one target rate R, built around an unchanged packed batch.
//
// The graph:
//   1. resample_map_kernel: per crop, validate the request in target terms and write the source span its outputs read,
//      clipped to the file, as request b of the inner packed batch (an invalid request as an invalid packed request, so
//      the packed batch's status and error word come out in crop order; an empty crop as the empty excerpt at N).
//   2. clx::launch_packed of the inner batch, as is: every span decoded to f32 along the columns of its [C, T] output.
//   3. resample_kernel: per (tile of outputs, crop, row), the tile's source samples staged in shared memory from the
//      packed output, then each output the dot product of its phase's coefficients with them.  Writes every element of
//      [n_crops * C, L], zeros included.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <numeric>

#include "claxon_b200.h"
#include "clx_internal.h"

namespace clx {

constexpr uint32_t RS_MAP_THREADS = 256;
constexpr uint32_t RS_THREADS = 256;
constexpr uint32_t RS_SMEM = 8192;      // source samples a CTA stages (32 KB)
constexpr uint32_t RS_MAX_TILE = 1024;  // outputs per CTA, 4 per thread
constexpr uint32_t RS_GROUP = 4;        // outputs of one phase per thread

__global__ void __launch_bounds__(RS_MAP_THREADS)
resample_map_kernel(CropCorpus cc, ResampleBuffers rs) {
    const uint32_t b = blockIdx.x * RS_MAP_THREADS + threadIdx.x;
    if (b == 0) *rs.count = rs.n_crops;
    if (b >= rs.n_crops) return;
    const clx_crop_request r = rs.requests[b];
    clx_packed_request q{0, 1, 0, 1};  // invalid (reserved != 0): status CLX_ERR_INVALID_ARGUMENT, nothing decoded
    ResamplePlan p{r.offset, 0, 0, 0, 0};
    int64_t len = 0;
    // Requests come from outside the program: nothing is read on behalf of one before it is known to be in range.
    if (r.reserved == 0 && r.file < cc.n_files && r.offset >= 0) {
        const uint32_t ti = rs.file_rate[r.file];
        const ResampleRate t = rs.rates[ti];
        const int64_t N = cc.file_len[r.file];
        const int64_t Nt = t.taps ? (int64_t)(((uint64_t)N * t.n + t.o - 1) / t.o) : N;  // (N < 2^36, n < 2^20)
        if (r.offset <= Nt) {
            len = (uint64_t)(Nt - r.offset) < rs.L ? Nt - r.offset : (int64_t)rs.L;
            p.rate = ti;
            p.ch = cc.file_ch[r.file];
            int64_t lo = N, hi = N;  // an empty crop: the valid empty excerpt at the file's end
            if (len > 0 && t.taps == 0) {
                lo = r.offset;
                hi = r.offset + len;
            } else if (len > 0) {  // blocks b0 .. b1 read x[b0 * o - w, b1 * o + w + o)
                const int64_t b0 = r.offset / t.n, b1 = (r.offset + len - 1) / t.n;
                lo = max(b0 * t.o - (int64_t)t.w, (int64_t)0);
                hi = min(b1 * t.o + t.w + t.o, N);
            }
            q = clx_packed_request{r.file, 0, lo, len > 0 ? hi - lo : -1};
            p.src_lo = lo;
            p.src_len = hi - lo;
        }
    }
    rs.excerpts[b] = q;
    rs.plan[b] = p;
    rs.lengths[b] = len;
}

// Grid: x over tiles of rs.tile outputs, y over the crops, z over the rows.  Source sample src_lo + i of crop b, row c
// is src[c * src_stride + starts[b] + i] for i < src_len; every other sample reads 0 (outside the file, by the span's
// construction).
__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(ResampleBuffers rs) {
    __shared__ float s_x[RS_SMEM];
    const uint32_t c = blockIdx.z;
    const uint64_t j0 = (uint64_t)blockIdx.x * rs.tile, je = min(j0 + rs.tile, rs.L);
    for (uint32_t b = blockIdx.y; b < rs.n_crops; b += gridDim.y) {
        const ResamplePlan p = rs.plan[b];
        float* row = rs.out + ((uint64_t)b * rs.C + c) * rs.L;
        const uint64_t len = c < p.ch ? (uint64_t)rs.lengths[b] : 0u;
        const uint64_t j1 = max(j0, min(je, len));  // outputs [j0, j1) computed, [j1, je) zero
        for (uint64_t j = j1 + threadIdx.x; j < je; j += RS_THREADS) row[j] = 0.f;
        if (j1 == j0) continue;
        const float* x = rs.src + (uint64_t)c * rs.src_stride + rs.starts[b];
        const ResampleRate t = rs.rates[p.rate];
        const uint32_t m = (uint32_t)(j1 - j0);
        if (t.taps == 0) {  // r == R: the span starts at the crop's offset
            for (uint32_t i = threadIdx.x; i < m; i += RS_THREADS) row[j0 + i] = x[j0 + i];
            continue;
        }
        const float* coefs = rs.coefs + t.coef;
        const int32_t* k0 = rs.k0 + t.k0;
        const uint64_t J0 = (uint64_t)p.offset + j0, blk0 = J0 / t.n;
        const uint32_t ph0 = (uint32_t)(J0 - blk0 * t.n);
        const uint64_t nblk = (J0 + m - 1) / t.n - blk0 + 1;  // the tile's blocks, blk0 .. blk0 + nblk - 1
        // Each thread computes one phase of RS_GROUP blocks g, g + G, g + 2G, ..., so that one coefficient load serves
        // RS_GROUP outputs; the tile reads x[blk0 * o - w, (blk0 + G * RS_GROUP) * o + w) of the file.
        const uint64_t G = (nblk + RS_GROUP - 1) / RS_GROUP;
        const int64_t s0 = (int64_t)(blk0 * t.o) - t.w - p.src_lo;
        const uint64_t span = G * RS_GROUP * t.o + 2ull * t.w;
        if (span <= RS_SMEM) {
            __syncthreads();  // the previous crop's reads of s_x are done
            for (uint32_t i = threadIdx.x; i < (uint32_t)span; i += RS_THREADS) {
                const int64_t a = s0 + i;
                s_x[i] = a >= 0 && a < p.src_len ? x[a] : 0.f;
            }
            __syncthreads();
            for (uint32_t u = threadIdx.x; u < (uint32_t)G * t.n; u += RS_THREADS) {
                const uint32_t g = u / t.n, ph = u - g * t.n;
                const float* h = coefs + ph;  // tap k at h[k * n]: lanes of consecutive phases read consecutive words
                const float* s = s_x + (g * t.o + t.w + k0[ph]);
                const uint32_t step = (uint32_t)G * t.o;
                float acc[RS_GROUP] = {};
#pragma unroll 2
                for (uint32_t k = 0; k < t.taps; k++) {
                    const float c = __ldg(h + (uint64_t)k * t.n);
#pragma unroll
                    for (uint32_t q = 0; q < RS_GROUP; q++) acc[q] = fmaf(c, s[q * step + k], acc[q]);
                }
#pragma unroll
                for (uint32_t q = 0; q < RS_GROUP; q++) {
                    const uint32_t rel = (g + q * (uint32_t)G) * t.n + ph;  // output j0 + rel - ph0
                    if (rel >= ph0 && rel - ph0 < m) row[j0 + rel - ph0] = acc[q];
                }
            }
        } else {  // a ratio too large to stage even a small tile: straight from the packed output
            for (uint32_t i = threadIdx.x; i < m; i += RS_THREADS) {
                const uint64_t rel = ph0 + i, blk = rel / t.n, ph = rel - blk * t.n;
                const float* h = coefs + ph;
                const int64_t a0 = s0 + (int64_t)(blk * t.o) + t.w + k0[ph];
                float acc = 0.f;
                for (uint32_t k = 0; k < t.taps; k++) {
                    const int64_t a = a0 + k;
                    acc = fmaf(__ldg(h + k * t.n), a >= 0 && a < p.src_len ? x[a] : 0.f, acc);
                }
                row[j0 + i] = acc;
            }
        }
    }
}

cudaError_t launch_resample_map(const CropCorpus& cc, const ResampleBuffers& rs, cudaStream_t stream, uint64_t* launches) {
    resample_map_kernel<<<(rs.n_crops + RS_MAP_THREADS - 1) / RS_MAP_THREADS, RS_MAP_THREADS, 0, stream>>>(cc, rs);
    (*launches)++;
    return cudaGetLastError();
}

cudaError_t launch_resample(const ResampleBuffers& rs, cudaStream_t stream, uint64_t* launches) {
    const dim3 grid((uint32_t)((rs.L + rs.tile - 1) / rs.tile), std::min<uint32_t>(rs.n_crops, 65535), rs.C);
    resample_kernel<<<grid, RS_THREADS, 0, stream>>>(rs);
    (*launches)++;
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side: the filter of each rate pair, in float64, stored as f32.

namespace {
struct Pair {
    uint64_t o, n, w;
    double base;
};

Pair pair_of(uint32_t r, uint32_t R) {
    const uint64_t g = std::gcd(r, R), o = r / g, n = R / g;
    const double base = (double)std::min(o, n) * 0.99;
    return {o, n, (uint64_t)std::ceil(6.0 * (double)o / base), base};
}

double tap_t(const Pair& p, uint64_t ph, int64_t k) { return ((double)k / (double)p.o - (double)ph / (double)p.n) * p.base; }

// The taps of phase ph with |t| < 6, [lo, hi] within [-w, w + o) (t grows with k; the k nearest ph * o / n has |t| <
// 0.5, so there is one at least).
void phase_taps(const Pair& p, uint64_t ph, int64_t* lo, int64_t* hi) {
    int64_t a = -(int64_t)p.w, e = (int64_t)(p.w + p.o);  // first k with t > -6
    while (a < e) {
        const int64_t m = a + (e - a) / 2;
        if (tap_t(p, ph, m) > -6.0) e = m;
        else a = m + 1;
    }
    *lo = a;
    e = (int64_t)(p.w + p.o);  // first k with t >= 6
    while (a < e) {
        const int64_t m = a + (e - a) / 2;
        if (tap_t(p, ph, m) >= 6.0) e = m;
        else a = m + 1;
    }
    *hi = a - 1;
}

uint64_t span_bound(const Pair& p, uint64_t L) {  // (the caller checks for overflow)
    return ((L - 1) / p.n + 2) * p.o + 2 * p.w;
}

bool span_overflows(const Pair& p, uint64_t L) {
    const uint64_t most = (UINT64_MAX - 2 * p.w) / p.o;  // blocks (w < 2^23, o < 2^20)
    return most < 2 || (L - 1) / p.n > most - 2;
}
}  // namespace

bool resample_tables(const uint32_t* file_rates, size_t n_files, uint32_t target, size_t num_frames, ResampleTables* t) {
    if (target == 0 || target > CLX_MAX_SAMPLE_RATE || num_frames == 0 || (!file_rates && n_files)) return false;
    constexpr uint64_t MAX_COEFS = 1ull << 24;
    std::vector<uint32_t> seen;  // the rate of each table
    t->file_rate.resize(n_files);
    t->bound = num_frames;
    for (size_t i = 0; i < n_files; i++) {
        const uint32_t r = file_rates[i];
        if (r == 0 || r > CLX_MAX_SAMPLE_RATE) return false;
        const size_t at = std::find(seen.begin(), seen.end(), r) - seen.begin();
        t->file_rate[i] = (uint32_t)at;
        if (at < seen.size()) continue;
        seen.push_back(r);
        if (r == target) {
            t->rates.push_back({1, 1, 0, 0, 0, 0});
            continue;
        }
        const Pair p = pair_of(r, target);
        if (p.n > MAX_COEFS - t->coefs.size()) return false;
        std::vector<int64_t> lo(p.n), hi(p.n);
        uint64_t taps = 0;
        for (uint64_t ph = 0; ph < p.n; ph++) {
            phase_taps(p, ph, &lo[ph], &hi[ph]);
            taps = std::max<uint64_t>(taps, hi[ph] - lo[ph] + 1);
        }
        if (taps > (MAX_COEFS - t->coefs.size()) / p.n) return false;
        if (span_overflows(p, num_frames)) return false;
        t->bound = std::max<uint64_t>(t->bound, span_bound(p, num_frames));
        const ResampleRate rr{(uint32_t)p.o, (uint32_t)p.n, (uint32_t)p.w, (uint32_t)taps, t->coefs.size(), t->k0.size()};
        t->coefs.resize(t->coefs.size() + p.n * taps, 0.f);
        for (uint64_t ph = 0; ph < p.n; ph++) {
            // taps k0 .. k0 + taps - 1, kept inside [-w, w + o) so that a tile's staged samples cover them; tap i of
            // phase ph at coef + i * n + ph
            const int64_t k0 = std::min<int64_t>(lo[ph], (int64_t)(p.w + p.o - taps));
            t->k0.push_back((int32_t)k0);
            for (int64_t k = lo[ph]; k <= hi[ph]; k++) {
                const double x = tap_t(p, ph, k), px = x * M_PI;
                const double sinc = x == 0.0 ? 1.0 : std::sin(px) / px, win = std::cos(x * M_PI / 12.0);
                t->coefs[rr.coef + (uint64_t)(k - k0) * p.n + ph] = (float)(sinc * win * win * p.base / (double)p.o);
            }
        }
        t->rates.push_back(rr);
    }
    // The largest tile (a power of two, at least 32) whose source samples fit in shared memory at every rate; a rate
    // that does not fit even then reads the packed output directly.
    t->tile = RS_MAX_TILE;
    for (const ResampleRate& r : t->rates)
        while (r.taps && t->tile > 32 && span_bound({r.o, r.n, r.w, 0.0}, t->tile + (RS_GROUP - 1) * r.n) > RS_SMEM)
            t->tile /= 2;
    return true;
}

}  // namespace clx

extern "C" size_t clx_resample_source_bound(uint32_t orig, uint32_t target, size_t num_frames) {
    if (orig == 0 || target == 0 || orig > CLX_MAX_SAMPLE_RATE || target > CLX_MAX_SAMPLE_RATE || num_frames == 0) return 0;
    if (orig == target) return num_frames;
    const clx::Pair p = clx::pair_of(orig, target);
    if (clx::span_overflows(p, num_frames)) return SIZE_MAX;
    return clx::span_bound(p, num_frames);
}
