// clx_scan.cuh — the one-CTA block scan of the packed planners: packed_scan_kernel (clx_crops.cu) and
// resample_packed_map_kernel (clx_resample.cu) lay excerpts out along columns with it.
#ifndef CLX_SCAN_CUH
#define CLX_SCAN_CUH
#include <cuda_runtime.h>
#include <stdint.h>

namespace clx {

constexpr uint32_t SCAN_THREADS = 1024;

// What packed_scan_kernel adds up: columns, slots, staging bytes and gather chunks.
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

}  // namespace clx
#endif
