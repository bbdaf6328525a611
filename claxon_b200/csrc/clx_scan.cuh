// clx_scan.cuh — the one-CTA block scan of the planners (clx_crops.cu, clx_resample.cu, clx_mel.cu), and the two
// layouts of a batch's excerpts that the crop and packed planners are templated on.
#ifndef CLX_SCAN_CUH
#define CLX_SCAN_CUH
#include <cuda_runtime.h>
#include <stdint.h>

#include "clx_internal.h"

namespace clx {

constexpr uint32_t SCAN_THREADS = 1024;

// What excerpt_scan_kernel adds up: columns, slots, staging bytes and gather chunks.
struct PackedSums {
    uint64_t cols, bytes;
    uint32_t slots, chunks;
    __device__ PackedSums operator+(const PackedSums& o) const {
        return {cols + o.cols, bytes + o.bytes, slots + o.slots, chunks + o.chunks};
    }
};

__device__ __forceinline__ PackedSums shfl_up(const PackedSums& x, uint32_t o) {
    return {__shfl_up_sync(0xffffffffu, x.cols, o), __shfl_up_sync(0xffffffffu, x.bytes, o),
            __shfl_up_sync(0xffffffffu, x.slots, o), __shfl_up_sync(0xffffffffu, x.chunks, o)};
}

// Exclusive scan of v over the CTA (SCAN_THREADS threads, all of them call it), after *carry; *carry then includes the
// whole CTA's sum.
__device__ __forceinline__ PackedSums cta_scan(PackedSums v, PackedSums* s_warp, PackedSums* carry) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    PackedSums x = v;
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const PackedSums y = shfl_up(x, o);
        if (lane >= o) x = x + y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        PackedSums w = s_warp[lane];
#pragma unroll
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const PackedSums y = shfl_up(w, o);
            if (lane >= o) w = w + y;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    const PackedSums before = *carry + (warp ? s_warp[warp - 1] : PackedSums{}) + x;
    const PackedSums excl{before.cols - v.cols, before.bytes - v.bytes, before.slots - v.slots, before.chunks - v.chunks};
    __syncthreads();
    if (threadIdx.x == SCAN_THREADS - 1) *carry = before;
    __syncthreads();
    return excl;
}

__host__ __device__ __forceinline__ uint64_t round_up_4(uint64_t x) { return (x + 3) & ~(uint64_t)3; }

// A request from outside the program, read as a packed request: nothing is read on its behalf before this holds.
__device__ __forceinline__ bool request_ok(const clx_packed_request& r, uint32_t n_files) {
    return r.reserved == 0 && r.file < n_files && r.offset >= 0 && r.length != 0 && r.length >= -1;
}
// Its excerpt of a file of N samples: min(length, N - offset) samples (N - offset for length -1); -1 for an offset past N.
__device__ __forceinline__ int64_t excerpt_length(const clx_packed_request& r, int64_t N) {
    if (r.offset > N) return -1;
    const int64_t rest = N - r.offset;
    return r.length == -1 || r.length > rest ? rest : r.length;
}

// The layouts: how request b reads and which excerpts a call uses; where excerpt b's output starts (start() in the
// scan, every thread of the CTA calling it, origin() afterwards) and whether it fits; what the zero pass clears for it
// on row c (b == n: after the excerpts) in elements of the output from row c's start; where unused slots decode to.
// Both write an excerpt's row c from origin + c * L.
struct CropLayout {  // crop b: rows [b * C, (b + 1) * C) of L columns, every crop used; the C trash rows after them
    const ExcerptBuffers& eb;
    __device__ uint32_t used() const { return eb.n; }
    __device__ clx_packed_request request(uint32_t b) const {
        const clx_crop_request r = eb.crop_requests[b];
        return {r.file, r.reserved, r.offset, (int64_t)eb.L};
    }
    __device__ uint64_t start(uint32_t, int64_t, PackedSums*, PackedSums*) const { return 0; }
    __device__ bool fits(uint64_t, int64_t) const { return true; }
    __device__ uint64_t origin(uint32_t b) const { return (uint64_t)b * eb.C * eb.L; }
    __device__ void zero(uint32_t b, uint32_t c, uint64_t* from, uint64_t* to) const {  // [covered, L)
        *from = *to = 0;
        if (b == eb.n) return;
        const uint64_t o = origin(b);
        *from = o + (c < eb.plan[b].ch ? (uint64_t)eb.lengths[b] : 0u);
        *to = o + eb.L;
    }
    __host__ __device__ uint64_t width() const { return eb.L; }  // the longest zero range
    __device__ uint64_t end(uint64_t, int64_t) const { return 0; }
    __device__ void set_end(uint64_t) const {}
    __device__ void keep_end() const {}
    __device__ uint64_t trash() const { return (uint64_t)eb.n * eb.C * eb.L; }
    __device__ uint64_t trash_width() const { return eb.L; }
};
struct PackedLayout {  // excerpt b: columns from starts[b] of rows 0 .. C - 1; the W trash columns after round_up_4(T)
    const ExcerptBuffers& eb;
    __device__ uint32_t used() const { return *eb.count; }
    __device__ clx_packed_request request(uint32_t b) const { return eb.packed_requests[b]; }
    // start_b: the scan of round_up_4(n_b) over the excerpts (n_b = 0 for the invalid ones), kept in starts[b]
    __device__ uint64_t start(uint32_t b, int64_t len, PackedSums* s_warp, PackedSums* s_cols) const {
        const uint64_t s = cta_scan(PackedSums{round_up_4((uint64_t)len), 0, 0, 0}, s_warp, s_cols).cols;
        if (b < eb.n) eb.starts[b] = (int64_t)s;
        return s;
    }
    __device__ bool fits(uint64_t start, int64_t len) const { return start + (uint64_t)len <= eb.T; }
    __device__ uint64_t origin(uint32_t b) const { return (uint64_t)eb.starts[b]; }
    // Excerpt b (that fits, n_b > 0): [start_b + n_b, start_b + round_up_4(n_b)) up to T on every row, and [start_b,
    // start_b + n_b) on rows its file does not have.  After the excerpts: [end, previous end).  Nothing else in [C, T]
    // was written by this call or the previous one.
    __device__ void zero(uint32_t b, uint32_t c, uint64_t* from, uint64_t* to) const {
        *from = *to = 0;
        if (b == eb.n) {
            *from = eb.end[0];
            *to = eb.end[1];
            return;
        }
        const uint64_t len = (uint64_t)eb.lengths[b];
        if (len == 0) return;
        const uint64_t start = origin(b), e = start + round_up_4(len);
        *from = start + (c < eb.plan[b].ch ? len : 0u);
        *to = e < eb.T ? e : eb.T;
    }
    __host__ __device__ uint64_t width() const { return eb.T; }
    // This call's end column: the furthest zero range of an excerpt that fits; the status pass makes it the previous one.
    __device__ uint64_t end(uint64_t start, int64_t len) const {
        const uint64_t e = start + round_up_4((uint64_t)len);
        return e < eb.T ? e : eb.T;
    }
    __device__ void set_end(uint64_t e) const { eb.end[0] = e; }
    __device__ void keep_end() const { eb.end[1] = eb.end[0]; }
    __device__ uint64_t trash() const { return round_up_4(eb.T); }
    __device__ uint64_t trash_width() const { return eb.L - round_up_4(eb.T); }
};

}  // namespace clx
#endif
