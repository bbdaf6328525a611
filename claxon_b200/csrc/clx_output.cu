// clx_output.cu — the output stage after the decode path: planar i32 (claxon's Block layout,
// reference src/frame.rs:477-481) -> interleaved little-endian samples of 2, 3 or 4 bytes, the form
// FlacSamples yields them in (src/lib.rs:473-519: for each inter-channel sample, every channel in turn),
// WAV writers store them in (examples/decode.rs:48-62) and the STREAMINFO MD5 is defined over
// (src/metadata.rs:52-53).  Runs on the device so that 16-bit audio crosses PCIe as 2 bytes per sample.
// Also planar i32 -> channels-first i32 / f32 rows, the [channels, samples] form of PyTorch audio code.
#include <cuda_runtime.h>
#include <stdint.h>

#include "claxon_b200.h"
#include "clx_internal.h"

namespace clx {

constexpr uint32_t IL_TILE = 4096;  // interleaved elements per CTA

// One CTA per (tile, frame).  Element i of a frame's interleaved block is sample t = i / n_channels of
// channel c = i % n_channels, i.e. planar element c * block_size + t.  Writes are coalesced; the reads
// are n_channels coalesced streams.  `sel` / `gate` (optional, see launch_interleave) restrict it to some frames.
template <int ESIZE>
__global__ void __launch_bounds__(256)
interleave_kernel(const clx_frame_desc* __restrict__ descs, uint32_t n_frames, const int32_t* __restrict__ planar,
                  uint8_t* __restrict__ dst, const uint8_t* __restrict__ sel, const int* __restrict__ gate) {
    if (gate != nullptr && *gate == 0) return;
    const uint32_t f = blockIdx.y;
    if (f >= n_frames || (sel != nullptr && sel[f] == 0)) return;
    const clx_frame_desc d = descs[f];
    const uint32_t nch = d.n_channels, bs = d.block_size, total = nch * bs;
    const uint32_t base = blockIdx.x * IL_TILE;
    if (base >= total) return;
    const int32_t* src = planar + d.out_offset;
    uint8_t* out = dst + d.out_offset * (uint64_t)ESIZE;
    if (ESIZE == 2 && nch == 2 && (d.out_offset & 1) == 0) {  // stereo 16-bit: one 4-byte store per sample pair
        for (uint32_t i = base / 2 + threadIdx.x; i < min(base + IL_TILE, total) / 2; i += 256) {
            const uint32_t l = (uint32_t)src[i] & 0xffffu, r = (uint32_t)src[bs + i];
            reinterpret_cast<uint32_t*>(out)[i] = l | (r << 16);
        }
        return;
    }
    for (uint32_t i = base + threadIdx.x; i < min(base + IL_TILE, total); i += 256) {
        const uint32_t t = i / nch, c = i - t * nch;
        const int32_t v = src[c * bs + t];
        if (ESIZE == 4) reinterpret_cast<int32_t*>(out)[i] = v;
        else if (ESIZE == 2) reinterpret_cast<int16_t*>(out)[i] = (int16_t)v;
        else {
            out[3 * (uint64_t)i] = (uint8_t)v;
            out[3 * (uint64_t)i + 1] = (uint8_t)(v >> 8);
            out[3 * (uint64_t)i + 2] = (uint8_t)(v >> 16);
        }
    }
}

// Channels-first: one CTA per (tile, frame) as above, over the frame's window only: samples [first, first + count) of
// each channel (wins[f] = first | count << 16).  Element i of the window is sample first + t of channel c (i = c * count
// + t), which goes to row c at element cols[f] + t of the buffer: reads and writes are coalesced along each row, and
// nothing outside the window is written.  F32: (float)s * 2^-(bits_per_sample - 1), rounded to nearest even, as the
// decode pass's channels flush.
template <bool F32>
__global__ void __launch_bounds__(256)
channels_kernel(const clx_frame_desc* __restrict__ descs, uint32_t n_frames, const int32_t* __restrict__ planar,
                int32_t* __restrict__ dst, const uint64_t* __restrict__ cols, uint64_t stride,
                const uint32_t* __restrict__ wins, const uint8_t* __restrict__ sel, const int* __restrict__ gate) {
    if (gate != nullptr && *gate == 0) return;
    const uint32_t f = blockIdx.y;
    if (f >= n_frames || (sel != nullptr && sel[f] == 0)) return;
    const clx_frame_desc d = descs[f];
    const uint32_t bs = d.block_size, first = wins[f] & 0xffffu, count = wins[f] >> 16;
    const uint32_t total = (uint32_t)d.n_channels * count;
    const uint32_t base = blockIdx.x * IL_TILE;
    if (base >= total) return;
    const int32_t* src = planar + d.out_offset + first;
    int32_t* out = dst + cols[f];
    const float scale = __int_as_float((int)(128u - d.bits_per_sample) << 23);  // 2^-(bps-1)
    for (uint32_t i = base + threadIdx.x; i < min(base + IL_TILE, total); i += 256) {
        const uint32_t c = i / count, t = i - c * count;
        const int32_t v = src[c * bs + t];
        out[c * stride + t] = F32 ? __float_as_int(__fmul_rn(__int2float_rn(v), scale)) : v;
    }
}

uint32_t output_elem_size(uint32_t mode) {
    return mode == CLX_OUT_INTERLEAVED_I16 ? 2u : mode == CLX_OUT_INTERLEAVED_I24 ? 3u : 4u;
}

cudaError_t launch_interleave(const clx_frame_desc* d_descs, uint32_t n_frames, uint32_t max_frame_elems, const int32_t* d_planar,
                              void* d_dst, uint32_t mode, cudaStream_t stream, uint64_t* launches, const uint8_t* sel,
                              const int* gate) {
    if (n_frames == 0 || mode == CLX_OUT_PLANAR_I32) return cudaSuccess;
    const uint32_t tiles = (max_frame_elems + IL_TILE - 1) / IL_TILE;
    for (uint32_t f0 = 0; f0 < n_frames; f0 += 65535) {  // gridDim.y limit
        const uint32_t nf = min(65535u, n_frames - f0);
        dim3 grid(tiles, nf);
        const uint8_t* s = sel ? sel + f0 : nullptr;
        if (mode == CLX_OUT_INTERLEAVED_I16)
            interleave_kernel<2><<<grid, 256, 0, stream>>>(d_descs + f0, nf, d_planar, (uint8_t*)d_dst, s, gate);
        else if (mode == CLX_OUT_INTERLEAVED_I24)
            interleave_kernel<3><<<grid, 256, 0, stream>>>(d_descs + f0, nf, d_planar, (uint8_t*)d_dst, s, gate);
        else
            interleave_kernel<4><<<grid, 256, 0, stream>>>(d_descs + f0, nf, d_planar, (uint8_t*)d_dst, s, gate);
    }
    (*launches)++;  // one pass, however many grids its frames need
    return cudaGetLastError();
}

cudaError_t launch_channels(const clx_frame_desc* d_descs, uint32_t n_frames, uint32_t max_frame_elems, const int32_t* d_planar,
                            void* d_dst, const uint64_t* d_cols, uint64_t stride, const uint32_t* d_wins, uint32_t mode,
                            cudaStream_t stream, uint64_t* launches, const uint8_t* sel, const int* gate) {
    if (n_frames == 0) return cudaSuccess;
    const uint32_t tiles = (max_frame_elems + IL_TILE - 1) / IL_TILE;
    for (uint32_t f0 = 0; f0 < n_frames; f0 += 65535) {  // gridDim.y limit
        const uint32_t nf = min(65535u, n_frames - f0);
        dim3 grid(tiles, nf);
        const uint8_t* s = sel ? sel + f0 : nullptr;
        if (mode == CLX_OUT_CHANNELS_F32)
            channels_kernel<true><<<grid, 256, 0, stream>>>(d_descs + f0, nf, d_planar, (int32_t*)d_dst, d_cols + f0, stride,
                                                            d_wins + f0, s, gate);
        else
            channels_kernel<false><<<grid, 256, 0, stream>>>(d_descs + f0, nf, d_planar, (int32_t*)d_dst, d_cols + f0, stride,
                                                            d_wins + f0, s, gate);
    }
    (*launches)++;  // one pass, however many grids its frames need
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
mark_status_kernel(const clx_frame_result* __restrict__ results, uint32_t n_frames, int32_t status, uint8_t* __restrict__ mark,
                   const int* __restrict__ gate) {
    if (*gate == 0) return;
    const uint32_t f = blockIdx.x * 256 + threadIdx.x;
    if (f < n_frames) mark[f] = results[f].status == status ? 1 : 0;
}

cudaError_t launch_mark_status(const clx_frame_result* d_results, uint32_t n_frames, int32_t status, uint8_t* d_mark,
                               const int* gate, cudaStream_t stream, uint64_t* launches) {
    if (n_frames == 0) return cudaSuccess;
    mark_status_kernel<<<(n_frames + 255) / 256, 256, 0, stream>>>(d_results, n_frames, status, d_mark, gate);
    (*launches)++;
    return cudaGetLastError();
}

}  // namespace clx
