// clx_resample.cu — resampled crop batches (include/claxon_b200.h, clx_batch_create_resampled_crops): [B, C, L] crops of
// a corpus whose files have different sample rates, all at one target rate R, built around an unchanged packed batch.
//
// The graph:
//   1. resample_map_kernel<CropLayout>: per crop, validate the request in target terms and write the source span its
//      outputs read, clipped to the file, as request b of the inner packed batch (an invalid request as an invalid
//      packed request, so the packed batch's status and error word come out in crop order; an empty crop as the empty
//      excerpt at N).
//   2. clx::launch_excerpts<PackedLayout> of the inner batch, as is: every span decoded to f32 along the columns of its
//      [C, T] output.
//   3. resample_kernel: per (tile of outputs, crop, row), the tile's source samples staged in shared memory from the
//      packed output, then each output the dot product of its phase's coefficients with them.  Writes every element of
//      [n_crops * C, L], zeros included.
// Resampled packed batches (clx_batch_create_resampled_packed) have the same graph over excerpts laid out along the
// columns of one [C, round_up_4(T)] output at rate R: resample_map_kernel<PackedLayout> (the layout, the fit and the
// source spans), the inner packed batch, and resample_packed_kernel, which runs resample_kernel's per-tile body on each
// excerpt's part of a tile of columns (CLX_RESAMPLE_TILE).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <numeric>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_scan.cuh"

namespace clx {

constexpr uint32_t RS_THREADS = 256;
constexpr uint32_t RS_SMEM = 8192;      // source samples a CTA stages (32 KB)
constexpr uint32_t RS_MAX_TILE = 1024;  // outputs per CTA, 4 per thread
constexpr uint32_t RS_GROUP = 4;        // outputs of one phase per thread

// The samples [lo, hi) of a file of N samples that outputs [offset, offset + len) at rate R read, clipped to the file;
// an empty excerpt (len 0) reads none, and is the valid empty excerpt at the file's end.
__device__ __forceinline__ void source_span(const ResampleRate& t, int64_t N, int64_t offset, int64_t len, int64_t* lo,
                                            int64_t* hi) {
    *lo = *hi = N;
    if (len > 0 && t.taps == 0) {
        *lo = offset;
        *hi = offset + len;
    } else if (len > 0) {  // blocks b0 .. b1 read x[b0 * o - w, b1 * o + w + o)
        const int64_t b0 = offset / t.n, b1 = (offset + len - 1) / t.n;
        *lo = max(b0 * t.o - (int64_t)t.w, (int64_t)0);
        *hi = min(b1 * t.o + t.w + t.o, N);
    }
}

// One CTA, SCAN_THREADS excerpts at a time: each request validated at rate R (N_t = ceil(N * n / o) in place of N) and
// its n_b taken, then the layout's start and fit (a packed batch's start_b is the scan of round_up_4(n_b) over the valid
// excerpts, and an excerpt fits when start_b + n_b <= T; a crop always fits).  One that fits becomes the packed request
// of its source span (an empty one, offset N_t, the valid empty excerpt at N); one that is invalid or does not fit
// becomes an invalid packed request in the same position, so the inner batch's status and error word come out in
// excerpt order, and a non-fit at R cannot reach the inner batch.
template <class Layout>
__global__ void __launch_bounds__(SCAN_THREADS)
resample_map_kernel(CropCorpus cc, ResampleBuffers rs, ExcerptBuffers eb) {
    __shared__ PackedSums s_warp[SCAN_THREADS / 32];
    __shared__ PackedSums s_cols;
    if (threadIdx.x == 0) s_cols = PackedSums{};
    __syncthreads();
    const Layout at{eb};
    const uint32_t n = eb.n, used = at.used();
    if (threadIdx.x == 0) *rs.count = used;
    for (uint32_t base = 0; base < n; base += SCAN_THREADS) {
        const uint32_t i = base + threadIdx.x;
        clx_packed_request r{0, 1, 0, 1};
        ResampleRate t{};
        int64_t N = 0, len = 0;
        bool valid = false;
        if (i < n && i < used) {  // (later excerpts are unused: length 0, an unused packed request)
            r = at.request(i);
            if (request_ok(r, cc.n_files)) {
                t = rs.rates[rs.file_rate[r.file]];
                N = cc.file_len[r.file];
                const int64_t Nt = t.taps ? (int64_t)(((uint64_t)N * t.n + t.o - 1) / t.o) : N;  // (N < 2^36, n < 2^20)
                len = excerpt_length(r, Nt);
                valid = len >= 0;
                if (!valid) len = 0;
            }
        }
        const uint64_t start = at.start(i, len, s_warp, &s_cols);
        const bool fit = valid && at.fits(start, len);
        clx_packed_request q{0, 1, 0, 1};  // invalid (reserved != 0): status CLX_ERR_INVALID_ARGUMENT, nothing decoded
        ResamplePlan p{0, 0, 0, 0, 0};
        if (fit) {
            int64_t lo, hi;
            source_span(t, N, r.offset, len, &lo, &hi);
            q = clx_packed_request{r.file, 0, lo, len > 0 ? hi - lo : -1};
            p = ResamplePlan{r.offset, lo, hi - lo, rs.file_rate[r.file], cc.file_ch[r.file]};
        }
        if (i < n) {
            rs.lengths[i] = fit ? len : 0;
            rs.plan[i] = p;
            rs.excerpts[i] = q;
        }
    }
}

// Outputs [j0, j0 + m) of one row of a crop or excerpt whose file has rate r != R, into row[j0 ..]: m <= the tile,
// p its ResamplePlan (offset: output 0's place in the file's resampled signal, src_lo / src_len: the decoded span), t
// its ResampleRate, x the span's row in the packed output; s_x the CTA's RS_SMEM floats of shared memory.  Every thread
// of the CTA runs it with the same arguments.  A macro rather than a function: that way resample_kernel compiles exactly
// as it did with the body written out, and resample_packed_kernel runs the same.
#define CLX_RESAMPLE_TILE(rs, t, p, x, row, j0, m, s_x)                                                                 \
    do {                                                                                                                \
        const float* coefs = rs.coefs + t.coef;                                                                         \
        const int32_t* k0 = rs.k0 + t.k0;                                                                               \
        const uint64_t J0 = (uint64_t)p.offset + j0, blk0 = J0 / t.n;                                                   \
        const uint32_t ph0 = (uint32_t)(J0 - blk0 * t.n);                                                               \
        const uint64_t nblk = (J0 + m - 1) / t.n - blk0 + 1; /* the tile's blocks, blk0 .. blk0 + nblk - 1 */           \
        /* Each thread computes one phase of RS_GROUP blocks g, g + G, g + 2G, ..., so that one coefficient load */     \
        /* serves RS_GROUP outputs; the tile reads x[blk0 * o - w, (blk0 + G * RS_GROUP) * o + w) of the file. */       \
        const uint64_t G = (nblk + RS_GROUP - 1) / RS_GROUP;                                                            \
        const int64_t s0 = (int64_t)(blk0 * t.o) - t.w - p.src_lo;                                                      \
        const uint64_t span = G * RS_GROUP * t.o + 2ull * t.w;                                                          \
        if (span <= RS_SMEM) {                                                                                          \
            __syncthreads(); /* the previous tile's reads of s_x are done */                                            \
            for (uint32_t i = threadIdx.x; i < (uint32_t)span; i += RS_THREADS) {                                       \
                const int64_t a = s0 + i;                                                                               \
                s_x[i] = a >= 0 && a < p.src_len ? x[a] : 0.f;                                                          \
            }                                                                                                           \
            __syncthreads();                                                                                            \
            for (uint32_t u = threadIdx.x; u < (uint32_t)G * t.n; u += RS_THREADS) {                                    \
                const uint32_t g = u / t.n, ph = u - g * t.n;                                                           \
                const float* h = coefs + ph; /* tap k at h[k * n]: lanes of consecutive phases read consecutive words */\
                const float* s = s_x + (g * t.o + t.w + k0[ph]);                                                        \
                const uint32_t step = (uint32_t)G * t.o;                                                                \
                float acc[RS_GROUP] = {};                                                                               \
                _Pragma("unroll 2") for (uint32_t k = 0; k < t.taps; k++) {                                             \
                    const float c = __ldg(h + (uint64_t)k * t.n);                                                       \
                    _Pragma("unroll") for (uint32_t q = 0; q < RS_GROUP; q++) acc[q] = fmaf(c, s[q * step + k], acc[q]);\
                }                                                                                                       \
                _Pragma("unroll") for (uint32_t q = 0; q < RS_GROUP; q++) {                                             \
                    const uint32_t rel = (g + q * (uint32_t)G) * t.n + ph; /* output j0 + rel - ph0 */                  \
                    if (rel >= ph0 && rel - ph0 < m) row[j0 + rel - ph0] = acc[q];                                      \
                }                                                                                                       \
            }                                                                                                           \
        } else { /* a ratio too large to stage even a small tile: straight from the packed output */                    \
            for (uint32_t i = threadIdx.x; i < m; i += RS_THREADS) {                                                    \
                const uint64_t rel = ph0 + i, blk = rel / t.n, ph = rel - blk * t.n;                                    \
                const float* h = coefs + ph;                                                                            \
                const int64_t a0 = s0 + (int64_t)(blk * t.o) + t.w + k0[ph];                                            \
                float acc = 0.f;                                                                                        \
                for (uint32_t k = 0; k < t.taps; k++) {                                                                 \
                    const int64_t a = a0 + k;                                                                           \
                    acc = fmaf(__ldg(h + k * t.n), a >= 0 && a < p.src_len ? x[a] : 0.f, acc);                          \
                }                                                                                                       \
                row[j0 + i] = acc;                                                                                      \
            }                                                                                                           \
        }                                                                                                               \
    } while (0)

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
        CLX_RESAMPLE_TILE(rs, t, p, x, row, j0, m, s_x);
    }
}

template <class Layout>
cudaError_t launch_resample_map(const CropCorpus& cc, const ResampleBuffers& rs, const ExcerptBuffers& eb,
                                cudaStream_t stream, uint64_t* launches) {
    resample_map_kernel<Layout><<<1, SCAN_THREADS, 0, stream>>>(cc, rs, eb);
    (*launches)++;
    return cudaGetLastError();
}
template cudaError_t launch_resample_map<CropLayout>(const CropCorpus&, const ResampleBuffers&, const ExcerptBuffers&,
                                                     cudaStream_t, uint64_t*);
template cudaError_t launch_resample_map<PackedLayout>(const CropCorpus&, const ResampleBuffers&, const ExcerptBuffers&,
                                                       cudaStream_t, uint64_t*);

cudaError_t launch_resample(const ResampleBuffers& rs, cudaStream_t stream, uint64_t* launches) {
    const dim3 grid((uint32_t)((rs.L + rs.tile - 1) / rs.tile), std::min<uint32_t>(rs.n_crops, 65535), rs.C);
    resample_kernel<<<grid, RS_THREADS, 0, stream>>>(rs);
    (*launches)++;
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Resampled packed batches (clx_batch_create_resampled_packed): rs as for crops, with n_crops = max_excerpts and L = the
// output's row stride; eb holds the caller's requests and count at rate R, and the target column starts.

// Grid: x over tiles of rs.tile columns, y over the rows.  The CTA of columns [c0, c0 + tile) walks the excerpts that
// overlap them, from the first one that ends after c0 (found by binary search: the ends start_b + n_b never decrease,
// since start_{b+1} >= start_b + n_b).  Each excerpt's segment is at most a tile, so it runs resample_kernel's per-tile
// body, or a copy at r == R; every other column of the range is written 0, so nothing is left from an earlier call.
// A tile of many short excerpts runs the body once per excerpt, each with its own staging and two barriers.
__global__ void __launch_bounds__(RS_THREADS)
resample_packed_kernel(ResampleBuffers rs, ExcerptBuffers eb) {
    __shared__ float s_x[RS_SMEM];
    const uint32_t c = blockIdx.y;
    const uint64_t c0 = (uint64_t)blockIdx.x * rs.tile, ce = min(c0 + rs.tile, rs.L);
    float* out = rs.out + (uint64_t)c * rs.L;
    const uint32_t used = min(*eb.count, rs.n_crops);
    uint32_t b = 0, e = used;
    while (b < e) {
        const uint32_t mid = (b + e) >> 1;
        if ((uint64_t)(eb.starts[mid] + rs.lengths[mid]) > c0) e = mid;
        else b = mid + 1;
    }
    uint64_t z = c0;  // columns [c0, z) are written
    for (; b < used; b++) {
        const uint64_t start = (uint64_t)eb.starts[b], len = (uint64_t)rs.lengths[b];
        if (start >= ce) break;
        if (len == 0) continue;
        const uint64_t lo = max(start, c0), hi = min(start + len, ce);
        for (uint64_t j = z + threadIdx.x; j < lo; j += RS_THREADS) out[j] = 0.f;
        z = hi;
        const ResamplePlan p = rs.plan[b];
        float* row = out + start;  // the excerpt's outputs j0 .. j0 + m - 1
        const uint64_t j0 = lo - start;
        const uint32_t m = (uint32_t)(hi - lo);
        if (c >= p.ch) {  // a row its file does not have
            for (uint32_t i = threadIdx.x; i < m; i += RS_THREADS) row[j0 + i] = 0.f;
            continue;
        }
        const float* x = rs.src + (uint64_t)c * rs.src_stride + rs.starts[b];
        const ResampleRate t = rs.rates[p.rate];
        if (t.taps == 0) {  // r == R: the span starts at the excerpt's offset
            for (uint32_t i = threadIdx.x; i < m; i += RS_THREADS) row[j0 + i] = x[j0 + i];
            continue;
        }
        CLX_RESAMPLE_TILE(rs, t, p, x, row, j0, m, s_x);
    }
    for (uint64_t j = z + threadIdx.x; j < ce; j += RS_THREADS) out[j] = 0.f;
}

cudaError_t launch_resample_packed(const ResampleBuffers& rs, const ExcerptBuffers& eb, cudaStream_t stream,
                                   uint64_t* launches) {
    const dim3 grid((uint32_t)((rs.L + rs.tile - 1) / rs.tile), rs.C);
    resample_packed_kernel<<<grid, RS_THREADS, 0, stream>>>(rs, eb);
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

// The inner packed batch's columns for excerpts that fit in T columns at rate R.  An excerpt of m >= 1 outputs reads a
// span of at most (floor((m - 1) / n) + 2) o + 2w <= (o / n) m + 2o + 2w samples, so round_up_4(span) <= (o / n) m + c
// with c = 2o + 2w + 3 (m + 3 when r == R, c = 3).  At most k = min(B, T) excerpts have outputs, and theirs add up to T
// at most: ceil(T * max o / n) + k * max c columns, rounded up to 4.  Accumulated rate by rate, in 128 bits.
struct SourceCols {
    unsigned __int128 per = 0;  // ceil(T * o / n), the largest so far
    uint64_t c = 0;             // the largest c so far
    void add(uint64_t o, uint64_t n, uint64_t w, bool same, uint64_t T) {
        const unsigned __int128 x = same ? (unsigned __int128)T : ((unsigned __int128)T * o + n - 1) / n;
        per = std::max(per, x);
        c = std::max<uint64_t>(c, same ? 3 : 2 * o + 2 * w + 3);
    }
    size_t total(uint64_t B, uint64_t T) const {  // SIZE_MAX on overflow
        const unsigned __int128 cols = per + (unsigned __int128)std::min(B, T) * c;
        return cols > SIZE_MAX - 3 ? SIZE_MAX : (size_t)((cols + 3) & ~(unsigned __int128)3);
    }
};
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

size_t resample_packed_bound(const ResampleTables& t, size_t max_excerpts, size_t max_samples) {
    SourceCols sc;
    for (const ResampleRate& r : t.rates) sc.add(r.o, r.n, r.w, r.taps == 0, max_samples);
    if (t.rates.empty()) sc.add(1, 1, 0, true, max_samples);
    return sc.total(max_excerpts, max_samples);
}

}  // namespace clx

extern "C" size_t clx_resample_source_bound(uint32_t orig, uint32_t target, size_t num_frames) {
    if (orig == 0 || target == 0 || orig > CLX_MAX_SAMPLE_RATE || target > CLX_MAX_SAMPLE_RATE || num_frames == 0) return 0;
    if (orig == target) return num_frames;
    const clx::Pair p = clx::pair_of(orig, target);
    if (clx::span_overflows(p, num_frames)) return SIZE_MAX;
    return clx::span_bound(p, num_frames);
}

extern "C" size_t clx_resample_packed_source_bound(const uint32_t* file_rates, size_t n_files, uint32_t target_rate,
                                                   size_t max_excerpts, size_t max_samples) {
    if (target_rate == 0 || target_rate > CLX_MAX_SAMPLE_RATE || max_excerpts == 0 || max_samples == 0 ||
        (!file_rates && n_files))
        return 0;
    clx::SourceCols sc;
    if (n_files == 0) sc.add(1, 1, 0, true, max_samples);
    for (size_t i = 0; i < n_files; i++) {
        const uint32_t r = file_rates[i];
        if (r == 0 || r > CLX_MAX_SAMPLE_RATE) return 0;
        const clx::Pair p = clx::pair_of(r, target_rate);
        sc.add(p.o, p.n, p.w, r == target_rate, max_samples);
    }
    return sc.total(max_excerpts, max_samples);
}
