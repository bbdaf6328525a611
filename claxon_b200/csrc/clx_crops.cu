// clx_crops.cu — crop batches (include/claxon_b200.h, clx_batch_create_crops): [B, C, L] excerpts of a corpus in device
// or pinned host memory, planned on the device inside the batch's graph; and packed batches (clx_batch_create_packed,
// after launch_crops), which lay variable-length excerpts along the columns of one [C, T] output with the same device
// code.
//
// The graph: the planner, then clx::launch_decode over every slot (with the device CRC-16), then the status pass.
//   1. crop_count_kernel: per crop, validate the request and binary-search the file's frame starts for the frames that
//      overlap [offset, min(offset + L, length)) (plan_range in claxon_b200/__init__.py does the same on the host).
//   2. crop_scan_kernel: one CTA, exclusive scan of the counts, so crops take consecutive slots in crop order and frames
//      in stream order (the device order of load_crops()'s windowed batch on a corpus of one shape).
//   2b. crop_gather_kernel, host corpora only: copies each crop's span of consecutive frames from mapped host memory
//      into its span of the batch's staging buffer, the layout load_crops() gathers on the host.
//   3. crop_emit_kernel: per slot, the frame's descriptor (out_offset = its place in the planar scratch; over a host
//      corpus, byte_offset = its place in the staging buffer), its column on the crop's first row and its window.  Slots
//      past the total go to the C trash rows after the output: up to the next multiple of 32 they repeat the last
//      planned frame, after that they get the filler frame, so fillers share warps only with each other; no window has
//      count 0.
//   4. crop_zero_kernel: zeroes exactly what no window of this call covers (columns past each crop's length, rows a
//      file does not have, every row of an invalid crop); the output is never cleared as a whole.
//   5. crop_status_kernel, after the decode: per crop the first failed slot, else the trailing-bytes verdict.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_scan.cuh"

namespace clx {

constexpr uint32_t CROP_THREADS = 256;

// The frames of a file, [f0, f1), that overlap its samples [lo, hi), lo < hi <= its length: the first of them in
// *first, their number returned (plan_range in claxon_b200/__init__.py does the same on the host).
__device__ __forceinline__ uint32_t overlapping_frames(const CropCorpus& cc, uint32_t f0, uint32_t f1, int64_t lo, int64_t hi,
                                                       uint32_t* first) {
    // the first frame that ends after lo: the one before the first later start above lo (else the last)
    uint32_t a = f0 + 1, e = f1;
    while (a < e) {
        const uint32_t m = (a + e) >> 1;
        if (cc.starts[m] > lo) e = m;
        else a = m + 1;
    }
    const uint32_t i0 = a - 1;
    // the frames that start before hi
    a = i0 + 1;
    e = f1;
    while (a < e) {
        const uint32_t m = (a + e) >> 1;
        if (cc.starts[m] >= hi) e = m;
        else a = m + 1;
    }
    *first = i0;
    return a - i0;
}

// The last b < n with scan[b] <= x, scan ascending: the owner of slot (or chunk) x (owners without any own none).
__device__ __forceinline__ uint32_t owner_of(const uint32_t* scan, uint32_t n, uint32_t x) {
    uint32_t a = 0, e = n;
    while (e - a > 1) {
        const uint32_t m = (a + e) >> 1;
        if (scan[m] <= x) a = m;
        else e = m;
    }
    return a;
}

__global__ void __launch_bounds__(CROP_THREADS)
crop_count_kernel(CropCorpus cc, CropBuffers cb) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b >= cb.n_crops) return;
    const clx_crop_request r = cb.requests[b];
    CropPlan p{r.offset, 0, 0, r.file, 0};
    int64_t len = 0;
    int32_t st = CLX_OK;
    // Requests come from outside the program: nothing is read on behalf of one before it is known to be in range.
    if (r.reserved != 0 || r.file >= cc.n_files || r.offset < 0 || r.offset > cc.file_len[r.file]) {
        st = CLX_ERR_INVALID_ARGUMENT;
        p.lo = 0;
        p.file = 0;
    } else {
        const uint32_t f0 = cc.file_frames[r.file], f1 = cc.file_frames[r.file + 1];
        const int64_t lo = r.offset, rest = cc.file_len[r.file] - lo;
        len = (uint64_t)rest < cb.L ? rest : (int64_t)cb.L;
        p.ch = cc.file_ch[r.file];
        if (len > 0)  // then the file has frames, and lo < its length
            p.count = min(overlapping_frames(cc, f0, f1, lo, lo + len, &p.first), cb.S);  // (never clipped: S bounds
                                                                                          // every count)
    }
    cb.plan[b] = p;
    cb.lengths[b] = len;
    cb.status[b] = st;
}

// Exclusive scan of the crops' counts into scan[0 .. n_crops), the total into scan[n_crops]; any n_crops, 1024 at a time.
__global__ void __launch_bounds__(SCAN_THREADS)
crop_scan_kernel(const CropPlan* __restrict__ plan, uint32_t n, uint32_t* __restrict__ scan) {
    __shared__ uint32_t s_warp[SCAN_THREADS / 32];
    __shared__ uint32_t s_carry;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += SCAN_THREADS) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < n ? plan[i].count : 0u;
        uint32_t x = v;
#pragma unroll
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = s_warp[lane];
#pragma unroll
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        const uint32_t excl = s_carry + (warp ? s_warp[warp - 1] : 0u) + x - v;
        if (i < n) scan[i] = excl;
        __syncthreads();
        if (threadIdx.x == SCAN_THREADS - 1) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) scan[n] = s_carry;
}

// Every load is a PCIe round trip of the order of a microsecond, so the grid keeps many in flight: a CTA copies
// GATHER_CHUNK bytes of one crop's span, each thread GATHER_VECS independent 16-byte loads before its stores.
constexpr uint32_t GATHER_THREADS = 256;
constexpr uint32_t GATHER_VECS = 4;
constexpr uint64_t GATHER_CHUNK = (uint64_t)GATHER_THREADS * GATHER_VECS * 16;

// Source bytes [s0, s1) of a host corpus go to staging[x + delta], where x + delta and x agree mod 16: 16-byte vectors
// between a scalar head and tail, copied by CTA `cx` of the `gx` CTAs given the span (the head and tail by cx 0).  A
// macro rather than a function: inlined as a function, the crop gather's loop-invariant values left the uniform
// datapath and the kernel lost a fifth of its rate; expanded, crop_gather_kernel compiles exactly as it did alone.
#define CLX_GATHER_SPAN(host_bytes, staging, s0, s1, delta, cx, gx)                                                     \
    do {                                                                                                                \
        uint64_t a = ((s0) + 15) & ~(uint64_t)15, e = (s1) & ~(uint64_t)15; /* the vector part [a, e) */               \
        if (e < a) a = e = (s1);                                             /* within one 16-byte block: all head */   \
        if ((cx) == 0 && threadIdx.x < 32) { /* head [s0, a) on threads 0-15, tail [e, s1) on 16-31 */                  \
            const uint64_t x = threadIdx.x < 16 ? (s0) + threadIdx.x : e + (threadIdx.x - 16);                          \
            if (x < (threadIdx.x < 16 ? a : (s1))) (staging)[x + (delta)] = (host_bytes)[x];                            \
        }                                                                                                               \
        const uint4* src = reinterpret_cast<const uint4*>((host_bytes) + a);                                            \
        uint4* dst = reinterpret_cast<uint4*>((staging) + (a + (delta)));                                               \
        const uint64_t n = (e - a) >> 4;                                                                                \
        for (uint64_t v = (uint64_t)(cx) * GATHER_THREADS * GATHER_VECS + threadIdx.x; v < n;                           \
             v += (uint64_t)(gx) * GATHER_THREADS * GATHER_VECS) {                                                      \
            uint4 r[GATHER_VECS];                                                                                       \
            _Pragma("unroll") for (uint32_t j = 0; j < GATHER_VECS; j++)                                                \
                if (v + j * GATHER_THREADS < n) r[j] = src[v + j * GATHER_THREADS];                                     \
            _Pragma("unroll") for (uint32_t j = 0; j < GATHER_VECS; j++)                                                \
                if (v + j * GATHER_THREADS < n) dst[v + j * GATHER_THREADS] = r[j];                                     \
        }                                                                                                               \
    } while (0)

// Grid: x over the chunks of a span, y over the crops.  Crop b's span [byte_offset(first), byte_offset(last) +
// byte_len(last)) goes to staging + b * span_stride + (start & 15).  Crops without frames copy nothing.
__global__ void __launch_bounds__(GATHER_THREADS)
crop_gather_kernel(CropCorpus cc, CropBuffers cb, uint8_t* __restrict__ staging) {
    for (uint32_t b = blockIdx.y; b < cb.n_crops; b += gridDim.y) {
        const CropPlan p = cb.plan[b];
        if (p.count == 0) continue;
        const uint64_t s0 = cc.descs[p.first].byte_offset;
        const clx_frame_desc& last = cc.descs[p.first + p.count - 1];
        const uint64_t s1 = last.byte_offset + last.byte_len;
        const uint64_t delta = (uint64_t)b * cc.span_stride + (s0 & 15) - s0;  // source byte x goes to staging[x + delta]
        CLX_GATHER_SPAN(cc.host_bytes, staging, s0, s1, delta, blockIdx.x, gridDim.x);
    }
}

// Where a batch puts excerpt b: its first column on row 0 (col), the staging address of its span's first byte b0 (span,
// host corpora), the filler frame's staging address, the trash columns and how many samples of a frame they take.
struct CropLayout {  // crop b: rows [b * C, (b + 1) * C) of L columns; the C trash rows after them
    const CropCorpus& cc;
    const CropBuffers& cb;
    __device__ uint64_t col(uint32_t b) const { return (uint64_t)b * cb.C * cb.L; }
    __device__ uint64_t span(uint32_t b, uint64_t b0) const { return (uint64_t)b * cc.span_stride + (b0 & 15); }
    __device__ uint64_t filler() const { return (uint64_t)cb.n_crops * cc.span_stride; }  // staged after the spans
    __device__ uint64_t trash() const { return (uint64_t)cb.n_crops * cb.C * cb.L; }
    __device__ uint64_t trash_width() const { return cb.L; }
};
struct PackedLayout {  // excerpt b: columns from starts[b] of rows 0 .. C - 1; the W trash columns after round_up_4(T)
    const CropCorpus& cc;
    const PackedBuffers& pb;
    __device__ uint64_t col(uint32_t b) const { return (uint64_t)pb.starts[b]; }
    __device__ uint64_t span(uint32_t b, uint64_t) const { return pb.stage[b]; }
    __device__ uint64_t filler() const { return cc.span_stride; }
    __device__ uint64_t trash() const { return (pb.T + 3) & ~(uint64_t)3; }
    __device__ uint64_t trash_width() const { return pb.W; }
};

// Slot s: the frame's descriptor (out_offset = its place in the planar scratch; over a host corpus, byte_offset = its
// place in the staging buffer), its column on row 0 and its window.
template <class Layout>
__device__ __forceinline__ void emit_slot(const CropCorpus& cc, const CropBuffers& cb, const Layout& at, uint32_t s,
                                          clx_frame_desc* descs, uint64_t* cols, uint32_t* wins) {
    const uint32_t total = cb.scan[cb.n_crops];
    const uint64_t trash = at.trash();
    clx_frame_desc d;
    uint64_t col;
    uint32_t win;
    // Unused slots in the last 32-slot group that holds planned frames repeat the last planned frame; the ones after it
    // get the filler frame.  Both go to the trash.  (The decode pass runs 32 frames per warp group: a filler next to
    // full-size frames takes the whole warp off its fast path, measured +1.1 ms per call at 176 400-sample crops.)
    const uint32_t slot = s < total ? s : s < ((total + 31) & ~31u) ? total - 1 : UINT32_MAX;
    if (slot == UINT32_MAX) {
        d = cc.descs[cc.n_frames];
        if (cc.span_stride) d.byte_offset = at.filler();  // staged there at creation
    } else {
        const uint32_t b = owner_of(cb.scan, cb.n_crops, slot);
        const CropPlan p = cb.plan[b];
        const uint32_t f = p.first + (slot - cb.scan[b]);
        d = cc.descs[f];
        if (cc.span_stride) {  // where the gather put the frame: its excerpt's span base plus its place in the span
            const uint64_t b0 = cc.descs[p.first].byte_offset;
            d.byte_offset = at.span(b, b0) + (d.byte_offset - b0);
        }
        const int64_t s0 = cc.starts[f], hi = p.lo + cb.lengths[b];
        const int64_t first = max(p.lo - s0, (int64_t)0);
        const int64_t count = min(s0 + (int64_t)d.block_size, hi) - s0 - first;
        col = at.col(b) + (uint64_t)(s0 + first - p.lo);
        win = (uint32_t)first | ((uint32_t)count << 16);
    }
    if (s >= total) {  // the whole frame (at most trash_width samples of it) on the trash
        col = trash;
        win = (uint32_t)(at.trash_width() < d.block_size ? at.trash_width() : d.block_size) << 16;
    }
    d.out_offset = (uint64_t)s * cb.slot_elems;
    descs[s] = d;
    cols[s] = col;
    wins[s] = win;
}

__global__ void __launch_bounds__(CROP_THREADS)
crop_emit_kernel(CropCorpus cc, CropBuffers cb, clx_frame_desc* __restrict__ descs, uint64_t* __restrict__ cols,
                 uint32_t* __restrict__ wins) {
    const uint32_t s = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (s >= cb.n_slots) return;
    emit_slot(cc, cb, CropLayout{cc, cb}, s, descs, cols, wins);
}

// One CTA row at a time (grid-stride over the n_crops * C output rows), its threads over the row's uncovered columns.
__global__ void __launch_bounds__(CROP_THREADS)
crop_zero_kernel(CropBuffers cb, int32_t* __restrict__ out) {
    const uint64_t rows = (uint64_t)cb.n_crops * cb.C;
    for (uint64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const uint32_t b = (uint32_t)(r / cb.C), c = (uint32_t)(r - (uint64_t)b * cb.C);
        const uint64_t covered = c < cb.plan[b].ch ? (uint64_t)cb.lengths[b] : 0u;
        int32_t* row = out + r * cb.L;
        for (uint64_t t = covered + blockIdx.y * CROP_THREADS + threadIdx.x; t < cb.L; t += (uint64_t)CROP_THREADS * gridDim.y)
            row[t] = 0;
    }
}

// Excerpt b's status after the decode: the planner's (an invalid request), else its first failed slot, else the
// trailing-bytes verdict; the error word keeps the smallest failure.
__device__ __forceinline__ void excerpt_status(const CropCorpus& cc, const CropBuffers& cb, uint32_t b,
                                               const clx_frame_result* results) {
    int32_t st = cb.status[b];
    unsigned long long kind = 0;
    if (st == CLX_OK) {
        const uint32_t s0 = cb.scan[b], s1 = cb.scan[b + 1];
        for (uint32_t s = s0; s < s1 && st == CLX_OK; s++) st = results[s].status;
        kind = 1;
        if (st == CLX_OK && s1 > s0) {  // an unconfirmed last frame inside the crop: what follows it
            const CropPlan p = cb.plan[b];
            const uint32_t last = cc.file_frames[p.file + 1] - 1;
            if (cc.file_tail[p.file] != CLX_OK && p.lo + cb.lengths[b] > cc.starts[last]) {
                st = cc.file_tail[p.file];
                kind = 2;
            }
        }
        cb.status[b] = st;
    }
    if (st != CLX_OK) atomicMin(cb.error, (kind << 62) | ((unsigned long long)b << 32) | (uint32_t)st);
}

__global__ void __launch_bounds__(CROP_THREADS)
crop_status_kernel(CropCorpus cc, CropBuffers cb, const clx_frame_result* __restrict__ results) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b >= cb.n_crops) return;
    excerpt_status(cc, cb, b, results);
}

cudaError_t launch_crops(const CropCorpus& cc, const CropBuffers& cb, const DecodeBuffers& db, const Plan& plan, bool crc,
                         cudaStream_t stream, uint64_t* launches) {
    cudaError_t e = cudaMemsetAsync(cb.error, 0xff, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const uint32_t crop_ctas = (cb.n_crops + CROP_THREADS - 1) / CROP_THREADS;
    crop_count_kernel<<<crop_ctas, CROP_THREADS, 0, stream>>>(cc, cb);
    crop_scan_kernel<<<1, SCAN_THREADS, 0, stream>>>(cb.plan, cb.n_crops, cb.scan);
    if (cc.host_bytes) {
        const dim3 ggrid((uint32_t)std::min<uint64_t>((cc.span_stride + GATHER_CHUNK - 1) / GATHER_CHUNK, 65535),
                         std::min<uint32_t>(cb.n_crops, 65535));
        crop_gather_kernel<<<ggrid, GATHER_THREADS, 0, stream>>>(cc, cb, const_cast<uint8_t*>(db.bytes));
        (*launches)++;
    }
    crop_emit_kernel<<<(cb.n_slots + CROP_THREADS - 1) / CROP_THREADS, CROP_THREADS, 0, stream>>>(
        cc, cb, const_cast<clx_frame_desc*>(db.descs), const_cast<uint64_t*>(db.cols), const_cast<uint32_t*>(db.wins));
    const uint64_t rows = (uint64_t)cb.n_crops * cb.C;
    const dim3 zgrid((uint32_t)std::min<uint64_t>(rows, 32768), (uint32_t)std::min<uint64_t>((cb.L + 8191) / 8192, 16));
    crop_zero_kernel<<<zgrid, CROP_THREADS, 0, stream>>>(cb, static_cast<int32_t*>(db.conv));
    *launches += 4;
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    e = launch_decode(db, plan, crc, stream, launches);
    if (e != cudaSuccess) return e;
    crop_status_kernel<<<crop_ctas, CROP_THREADS, 0, stream>>>(cc, cb, db.results);
    (*launches)++;
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Packed batches (clx_batch_create_packed): the same graph over variable-length excerpts laid out along the columns of
// one [C, stride] output.  packed_count_kernel validates and searches like crop_count_kernel; packed_scan_kernel gives
// the column starts, decides which excerpts fit, and scans their slots, staging bytes and gather chunks; the gather,
// emit and status bodies are the crop batch's; packed_zero_kernel zeroes the uncovered part of each excerpt's columns
// and the columns between this call's end and the previous call's.

__global__ void __launch_bounds__(CROP_THREADS)
packed_count_kernel(CropCorpus cc, CropBuffers cb, PackedBuffers pb) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b >= cb.n_crops) return;
    CropPlan p{0, 0, 0, 0, 0};
    int64_t len = 0;
    int32_t st = CLX_OK;
    if (b < *pb.count) {  // (later excerpts are unused: status CLX_OK, length 0, no frames)
        const clx_packed_request r = pb.requests[b];
        if (r.reserved != 0 || r.file >= cc.n_files || r.offset < 0 || r.offset > cc.file_len[r.file] || r.length == 0 ||
            r.length < -1) {
            st = CLX_ERR_INVALID_ARGUMENT;
        } else {
            const int64_t rest = cc.file_len[r.file] - r.offset;
            len = r.length == -1 || r.length > rest ? rest : r.length;
            p = CropPlan{r.offset, 0, 0, r.file, cc.file_ch[r.file]};
            if (len > 0)
                p.count = overlapping_frames(cc, cc.file_frames[r.file], cc.file_frames[r.file + 1], r.offset, r.offset + len,
                                             &p.first);
        }
    }
    cb.plan[b] = p;
    cb.lengths[b] = len;
    cb.status[b] = st;
}

// One CTA, SCAN_THREADS excerpts at a time.  Columns first: start_b is the scan of round_up_4(n_b) over the valid
// excerpts, and an excerpt fits when start_b + n_b <= T.  Then the slots of the excerpts that fit; one whose slots would
// pass n_slots does not fit either (never the case: n_slots is clx_packed_frames_bound; this keeps every later write in
// bounds whatever the requests).  Both rules leave the excerpts that fit a prefix of the valid ones.  Over a host corpus,
// each excerpt that fits and has frames takes span + 15 staging bytes, its span starting at the first address of the
// same residue mod 16 as its source, and ceil(span / GATHER_CHUNK) gather chunks.
__global__ void __launch_bounds__(SCAN_THREADS)
packed_scan_kernel(CropCorpus cc, CropBuffers cb, PackedBuffers pb) {
    __shared__ PackedSums s_warp[SCAN_THREADS / 32];
    __shared__ PackedSums s_cols, s_slots, s_final;
    __shared__ unsigned long long s_end;
    if (threadIdx.x == 0) s_cols = s_slots = s_final = PackedSums{}, s_end = 0;
    __syncthreads();
    const uint32_t n = cb.n_crops, used = *pb.count;
    for (uint32_t base = 0; base < n; base += SCAN_THREADS) {
        const uint32_t i = base + threadIdx.x;
        const bool valid = i < n && i < used && cb.status[i] == CLX_OK;
        const int64_t len = valid ? cb.lengths[i] : 0;
        const uint64_t cols = ((uint64_t)len + 3) & ~(uint64_t)3;
        const uint64_t start = cta_scan(PackedSums{cols, 0, 0, 0}, s_warp, &s_cols).cols;
        bool fit = valid && start + (uint64_t)len <= pb.T;
        const CropPlan p = i < n ? cb.plan[i] : CropPlan{};
        const uint32_t k = fit ? p.count : 0u;
        const uint32_t slot0 = cta_scan(PackedSums{0, 0, k, 0}, s_warp, &s_slots).slots;  // (every thread scans)
        fit = fit && slot0 + k <= cb.n_slots;
        uint64_t span = 0, s0 = 0;
        if (fit && p.count && cc.host_bytes) {
            s0 = cc.descs[p.first].byte_offset;
            const clx_frame_desc& last = cc.descs[p.first + p.count - 1];
            span = last.byte_offset + last.byte_len - s0;
        }
        const PackedSums mine{0, span ? span + 15 : 0, fit ? p.count : 0u,
                              span ? (uint32_t)((span + GATHER_CHUNK - 1) / GATHER_CHUNK) : 0u};
        const PackedSums at = cta_scan(mine, s_warp, &s_final);
        if (i < n) {
            pb.starts[i] = (int64_t)start;
            cb.scan[i] = at.slots;
            pb.chunks[i] = at.chunks;
            pb.stage[i] = at.bytes + ((s0 - at.bytes) & 15);
            if (valid && !fit) {
                cb.status[i] = CLX_ERR_INVALID_ARGUMENT;
                cb.lengths[i] = 0;
            }
            if (fit && len > 0) atomicMax(&s_end, (unsigned long long)(start + cols < pb.T ? start + cols : pb.T));
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        cb.scan[n] = s_final.slots;
        pb.chunks[n] = s_final.chunks;
        pb.end[0] = s_end;
    }
}

// Grid-stride over the chunks of every span: chunk k belongs to the excerpt whose chunk range holds it.
__global__ void __launch_bounds__(GATHER_THREADS)
packed_gather_kernel(CropCorpus cc, CropBuffers cb, PackedBuffers pb, uint8_t* __restrict__ staging) {
    const uint32_t total = pb.chunks[cb.n_crops];
    for (uint32_t k = blockIdx.x; k < total; k += gridDim.x) {
        const uint32_t b = owner_of(pb.chunks, cb.n_crops, k);
        const CropPlan p = cb.plan[b];
        const uint64_t s0 = cc.descs[p.first].byte_offset;
        const clx_frame_desc& last = cc.descs[p.first + p.count - 1];
        const uint64_t s1 = last.byte_offset + last.byte_len, delta = pb.stage[b] - s0;
        const uint32_t cx = k - pb.chunks[b], gx = pb.chunks[b + 1] - pb.chunks[b];
        CLX_GATHER_SPAN(cc.host_bytes, staging, s0, s1, delta, cx, gx);
    }
}

__global__ void __launch_bounds__(CROP_THREADS)
packed_emit_kernel(CropCorpus cc, CropBuffers cb, PackedBuffers pb, clx_frame_desc* __restrict__ descs,
                   uint64_t* __restrict__ cols, uint32_t* __restrict__ wins) {
    const uint32_t s = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (s >= cb.n_slots) return;
    emit_slot(cc, cb, PackedLayout{cc, pb}, s, descs, cols, wins);
}

// Rows (b, c) of the excerpts, then C rows for the tail.  Excerpt b (that fits, n_b > 0): columns [start_b + n_b,
// start_b + round_up_4(n_b)) up to T on every row, and [start_b, start_b + n_b) on rows its file does not have.  Tail:
// [end, previous end) on every row.  Nothing else in [C, T] was written by this call or the previous one.
__global__ void __launch_bounds__(CROP_THREADS)
packed_zero_kernel(CropBuffers cb, PackedBuffers pb, int32_t* __restrict__ out) {
    const uint64_t rows = (uint64_t)(cb.n_crops + 1) * cb.C;
    for (uint64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const uint32_t b = (uint32_t)(r / cb.C), c = (uint32_t)(r - (uint64_t)b * cb.C);
        uint64_t from, to;
        if (b == cb.n_crops) {
            from = pb.end[0];
            to = pb.end[1];
        } else {
            const uint64_t len = (uint64_t)cb.lengths[b], start = (uint64_t)pb.starts[b];
            if (len == 0) continue;
            from = start + (c < cb.plan[b].ch ? len : 0u);
            to = start + ((len + 3) & ~(uint64_t)3);
            if (to > pb.T) to = pb.T;
        }
        int32_t* row = out + c * cb.L;
        for (uint64_t t = from + blockIdx.y * CROP_THREADS + threadIdx.x; t < to; t += (uint64_t)CROP_THREADS * gridDim.y)
            row[t] = 0;
    }
}

// After the decode: each excerpt's status, and this call's end column becomes the previous one for the next call.
__global__ void __launch_bounds__(CROP_THREADS)
packed_status_kernel(CropCorpus cc, CropBuffers cb, PackedBuffers pb, const clx_frame_result* __restrict__ results) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b == 0) pb.end[1] = pb.end[0];
    if (b >= cb.n_crops) return;
    excerpt_status(cc, cb, b, results);
}

cudaError_t launch_packed(const CropCorpus& cc, const CropBuffers& cb, const PackedBuffers& pb, const DecodeBuffers& db,
                          const Plan& plan, bool crc, cudaStream_t stream, uint64_t* launches) {
    cudaError_t e = cudaMemsetAsync(cb.error, 0xff, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const uint32_t ctas = (cb.n_crops + CROP_THREADS - 1) / CROP_THREADS;
    packed_count_kernel<<<ctas, CROP_THREADS, 0, stream>>>(cc, cb, pb);
    packed_scan_kernel<<<1, SCAN_THREADS, 0, stream>>>(cc, cb, pb);
    if (cc.host_bytes) {
        packed_gather_kernel<<<pb.max_chunks, GATHER_THREADS, 0, stream>>>(cc, cb, pb, const_cast<uint8_t*>(db.bytes));
        (*launches)++;
    }
    packed_emit_kernel<<<(cb.n_slots + CROP_THREADS - 1) / CROP_THREADS, CROP_THREADS, 0, stream>>>(
        cc, cb, pb, const_cast<clx_frame_desc*>(db.descs), const_cast<uint64_t*>(db.cols), const_cast<uint32_t*>(db.wins));
    const uint64_t rows = (uint64_t)(cb.n_crops + 1) * cb.C;
    const dim3 zgrid((uint32_t)std::min<uint64_t>(rows, 32768), (uint32_t)std::min<uint64_t>((pb.T + 8191) / 8192, 16));
    packed_zero_kernel<<<zgrid, CROP_THREADS, 0, stream>>>(cb, pb, static_cast<int32_t*>(db.conv));
    *launches += 4;
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    e = launch_decode(db, plan, crc, stream, launches);
    if (e != cudaSuccess) return e;
    packed_status_kernel<<<ctas, CROP_THREADS, 0, stream>>>(cc, cb, pb, db.results);
    (*launches)++;
    return cudaGetLastError();
}

// The filler frame (FLAC frame header, src/frame.rs:131-316): sync 0xFFF8 (fixed blocking); block size code 1 (192
// samples), sample rate code 0 (from STREAMINFO); channel assignment 0 (one channel), sample size code 4 (16 bits); frame
// number 0; CRC-8.  One CONSTANT subframe (type 0, no wasted bits) of value 0 in 16 bits, then the CRC-16.
size_t filler_frame(uint8_t* out, size_t cap) {
    uint8_t f[11] = {0xff, 0xf8, 0x10, 0x08, 0x00, 0, 0x00, 0x00, 0x00, 0, 0};
    f[5] = clx_crc8(f, 5);
    const uint16_t crc = clx_crc16(f, 9);
    f[9] = (uint8_t)(crc >> 8);
    f[10] = (uint8_t)crc;
    if (out && cap >= sizeof f) memcpy(out, f, sizeof f);
    return sizeof f;
}

}  // namespace clx

extern "C" {

size_t clx_crop_filler_frame(uint8_t* out, size_t cap) { return clx::filler_frame(out, cap); }

size_t clx_crop_frames_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                             size_t num_frames) {
    if (num_frames == 0 || !file_frames || (!descs && n_frames) || file_frames[n_files] != n_frames) return 0;
    for (size_t i = 0; i < n_files; i++)
        if (file_frames[i + 1] < file_frames[i]) return 0;
    uint32_t m = 0;  // smallest block size of a frame that is not the last of its file (0: none)
    size_t most = 0;  // frames of the largest file
    for (size_t i = 0; i < n_files; i++) {
        most = std::max<size_t>(most, file_frames[i + 1] - file_frames[i]);
        for (size_t f = file_frames[i]; f + 1 < file_frames[i + 1]; f++)
            if (m == 0 || descs[f].block_size < m) m = descs[f].block_size;
    }
    if (m == 0 || num_frames == 1) return 1;
    // k overlapping frames: the first and the last give at least one sample each, the k - 2 between them whole blocks
    const size_t s = (num_frames - 2) / m + 2;
    return std::max<size_t>(1, std::min(s, most));
}

size_t clx_crop_bytes_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                            size_t num_frames) {
    const size_t S = clx_crop_frames_bound(descs, n_frames, file_frames, n_files, num_frames);
    if (S == 0) return 0;
    uint64_t most = 0;
    for (size_t i = 0; i < n_files; i++)  // a crop from frame f spans f .. min(f + S, end of its file) - 1
        for (size_t f = file_frames[i]; f < file_frames[i + 1]; f++) {
            const clx_frame_desc& last = descs[std::min<size_t>(f + S, file_frames[i + 1]) - 1];
            const uint64_t end = last.byte_offset + last.byte_len;
            if (end > descs[f].byte_offset) most = std::max<uint64_t>(most, end - descs[f].byte_offset);
        }
    return most;
}

size_t clx_packed_frames_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                               size_t max_excerpts, size_t max_samples) {
    if (max_excerpts == 0 || max_samples == 0 || !file_frames || (!descs && n_frames) || file_frames[n_files] != n_frames)
        return 0;
    for (size_t i = 0; i < n_files; i++)
        if (file_frames[i + 1] < file_frames[i]) return 0;
    uint32_t m = 0;   // smallest block size of a frame that is not the last of its file (0: none)
    size_t most = 0;  // frames of the largest file
    for (size_t i = 0; i < n_files; i++) {
        most = std::max<size_t>(most, file_frames[i + 1] - file_frames[i]);
        for (size_t f = file_frames[i]; f + 1 < file_frames[i + 1]; f++)
            if (m == 0 || descs[f].block_size < m) m = descs[f].block_size;
    }
    // Excerpts that fit hold at most T samples in all, so at most k = min(B, T) of them have frames.  One of n samples
    // overlaps at most (n - 2) / m + 2 frames (the first and last give one sample or more, the ones between whole non-last
    // blocks; 1 <= 2 - 1 / m for n = 1), so all of them together floor((T - 2k) / m) + 2k, since the sum grows with k.
    const size_t k = std::min(max_excerpts, max_samples);
    if (m == 0) return k;
    const int64_t d = (int64_t)max_samples - 2 * (int64_t)k;  // (>= -T: no overflow)
    const int64_t q = d >= 0 ? d / m : -((-d + m - 1) / (int64_t)m);
    const size_t s = (size_t)(q + 2 * (int64_t)k);
    return std::max<size_t>(1, most && k <= SIZE_MAX / most ? std::min(s, k * most) : s);
}

size_t clx_packed_bytes_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                              size_t max_excerpts, size_t max_samples) {
    const size_t S = clx_packed_frames_bound(descs, n_frames, file_frames, n_files, max_excerpts, max_samples);
    if (S == 0) return 0;
    // An excerpt's span, frames f .. g of one file: the advances from f to g plus byte_len(g), at most its frame count
    // times the largest per-frame advance (gaps between frames included), so every span together at most S times it.
    uint64_t adv = 0;
    for (size_t i = 0; i < n_files; i++)
        for (size_t f = file_frames[i]; f < file_frames[i + 1]; f++) {
            adv = std::max<uint64_t>(adv, descs[f].byte_len);
            if (f + 1 < file_frames[i + 1] && descs[f + 1].byte_offset > descs[f].byte_offset)
                adv = std::max<uint64_t>(adv, descs[f + 1].byte_offset - descs[f].byte_offset);
        }
    if (max_excerpts > SIZE_MAX / 32 || (adv && S > (SIZE_MAX - 16 * max_excerpts) / adv)) return SIZE_MAX;
    return S * adv + 16 * max_excerpts;
}

}  // extern "C"
