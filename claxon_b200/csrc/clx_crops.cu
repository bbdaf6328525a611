// clx_crops.cu — crop batches (include/claxon_b200.h, clx_batch_create_crops): [B, C, L] excerpts of a corpus in device
// or pinned host memory, planned on the device inside the batch's graph.
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

namespace clx {

constexpr uint32_t CROP_THREADS = 256;
constexpr uint32_t SCAN_THREADS = 1024;

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
        if (len > 0) {  // then the file has frames, and lo < its length
            const int64_t hi = lo + len;
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
            p.first = i0;
            p.count = min(a - i0, cb.S);  // (never clipped: S bounds every count, see clx_crop_frames_bound)
        }
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

// Grid: x over the chunks of a span, y over the crops.  Crop b's span [byte_offset(first), byte_offset(last) +
// byte_len(last)) goes to staging + b * span_stride + (start & 15): source and destination agree mod 16, so the body is
// 16-byte vectors between a scalar head and tail.  Crops without frames copy nothing.
__global__ void __launch_bounds__(GATHER_THREADS)
crop_gather_kernel(CropCorpus cc, CropBuffers cb, uint8_t* __restrict__ staging) {
    for (uint32_t b = blockIdx.y; b < cb.n_crops; b += gridDim.y) {
        const CropPlan p = cb.plan[b];
        if (p.count == 0) continue;
        const uint64_t s0 = cc.descs[p.first].byte_offset;
        const clx_frame_desc& last = cc.descs[p.first + p.count - 1];
        const uint64_t s1 = last.byte_offset + last.byte_len;
        const uint64_t delta = (uint64_t)b * cc.span_stride + (s0 & 15) - s0;  // source byte x goes to staging[x + delta]
        uint64_t a = (s0 + 15) & ~(uint64_t)15, e = s1 & ~(uint64_t)15;      // the vector part [a, e)
        if (e < a) a = e = s1;                                                // within one 16-byte block: all head
        if (blockIdx.x == 0 && threadIdx.x < 32) {  // head [s0, a) on threads 0-15, tail [e, s1) on 16-31
            const uint64_t x = threadIdx.x < 16 ? s0 + threadIdx.x : e + (threadIdx.x - 16);
            if (x < (threadIdx.x < 16 ? a : s1)) staging[x + delta] = cc.host_bytes[x];
        }
        const uint4* src = reinterpret_cast<const uint4*>(cc.host_bytes + a);
        uint4* dst = reinterpret_cast<uint4*>(staging + (a + delta));
        const uint64_t n = (e - a) >> 4;
        for (uint64_t v = (uint64_t)blockIdx.x * GATHER_THREADS * GATHER_VECS + threadIdx.x; v < n;
             v += (uint64_t)gridDim.x * GATHER_THREADS * GATHER_VECS) {
            uint4 r[GATHER_VECS];
#pragma unroll
            for (uint32_t j = 0; j < GATHER_VECS; j++)
                if (v + j * GATHER_THREADS < n) r[j] = src[v + j * GATHER_THREADS];
#pragma unroll
            for (uint32_t j = 0; j < GATHER_VECS; j++)
                if (v + j * GATHER_THREADS < n) dst[v + j * GATHER_THREADS] = r[j];
        }
    }
}

__global__ void __launch_bounds__(CROP_THREADS)
crop_emit_kernel(CropCorpus cc, CropBuffers cb, clx_frame_desc* __restrict__ descs, uint64_t* __restrict__ cols,
                 uint32_t* __restrict__ wins) {
    const uint32_t s = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (s >= cb.n_slots) return;
    const uint32_t total = cb.scan[cb.n_crops];
    const uint64_t trash = (uint64_t)cb.n_crops * cb.C * cb.L;  // the rows after the output
    clx_frame_desc d;
    uint64_t col;
    uint32_t win;
    // Unused slots in the last 32-slot group that holds planned frames repeat the last planned frame; the ones after it
    // get the filler frame.  Both go to the trash rows.  (The decode pass runs 32 frames per warp group: a filler next to
    // full-size frames takes the whole warp off its fast path, measured +1.1 ms per call at 176 400-sample crops.)
    const uint32_t slot = s < total ? s : s < ((total + 31) & ~31u) ? total - 1 : UINT32_MAX;
    if (slot == UINT32_MAX) {
        d = cc.descs[cc.n_frames];
        if (cc.span_stride) d.byte_offset = (uint64_t)cb.n_crops * cc.span_stride;  // staged after the spans at creation
    } else {
        // the crop that owns the slot: the last b with scan[b] <= slot (crops without frames own no slot)
        uint32_t a = 0, e = cb.n_crops;
        while (e - a > 1) {
            const uint32_t m = (a + e) >> 1;
            if (cb.scan[m] <= slot) a = m;
            else e = m;
        }
        const uint32_t b = a;
        const CropPlan p = cb.plan[b];
        const uint32_t f = p.first + (slot - cb.scan[b]);
        d = cc.descs[f];
        if (cc.span_stride) {  // where crop_gather_kernel put the frame: its crop's span base plus its place in the span
            const uint64_t b0 = cc.descs[p.first].byte_offset;
            d.byte_offset = (uint64_t)b * cc.span_stride + (b0 & 15) + (d.byte_offset - b0);
        }
        const int64_t s0 = cc.starts[f], hi = p.lo + cb.lengths[b];
        const int64_t first = max(p.lo - s0, (int64_t)0);
        const int64_t count = min(s0 + (int64_t)d.block_size, hi) - s0 - first;
        col = (uint64_t)b * cb.C * cb.L + (uint64_t)(s0 + first - p.lo);
        win = (uint32_t)first | ((uint32_t)count << 16);
    }
    if (s >= total) {  // the whole frame (at most L samples of it) on the trash rows
        col = trash;
        win = (uint32_t)(cb.L < d.block_size ? cb.L : d.block_size) << 16;
    }
    d.out_offset = (uint64_t)s * cb.slot_elems;
    descs[s] = d;
    cols[s] = col;
    wins[s] = win;
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

__global__ void __launch_bounds__(CROP_THREADS)
crop_status_kernel(CropCorpus cc, CropBuffers cb, const clx_frame_result* __restrict__ results) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b >= cb.n_crops) return;
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

}  // extern "C"
