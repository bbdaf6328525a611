// clx_internal.h — shared between the kernels (clx_decode.cu) and the C ABI (clx_api.cu).
#ifndef CLX_INTERNAL_H
#define CLX_INTERNAL_H
#include <cuda_runtime.h>
#include <stdint.h>
#include "claxon_b200.h"

// Device-only marker: the frame has an LPC order above what the first kernel instance keeps in
// registers and must be decoded by the 32-tap instance.  Never returned through the C ABI.
#define CLX_INTERNAL_NEED_HIGH_ORDER (-1)
// Device-only marker: the cooperative kernel declined the frame (anything irregular: malformed
// input, escape codes, oversize frames ...); the generic lane-per-frame kernel decodes it.
// Returned through the C ABI only under CLX_OPT_NO_GENERIC (the generic kernel then does not run).
#define CLX_INTERNAL_NEED_GENERIC (-2)
// Device-only marker of the throughput path: decode the frame again with the i64 accumulator (clx_fused.cu).
// Returned through the C ABI only under CLX_OPT_NO_WIDE (the second chance then does not run).
#define CLX_INTERNAL_NEED_WIDE (-3)

namespace clx {
struct CoopPlan {          // whether / how a batch uses the fast path
    uint32_t G = 0;             // 0: generic kernel only; 1: warp per frame (clx_coop.cu); 2: lane per frame index pass + lane per subframe decode pass (clx_fused.cu)
    uint32_t frame_stride = 0;
    uint32_t channels = 0;      // channel slots per frame (power of two >= max channels in the batch)
    size_t smem_bytes = 0;
    uint32_t max_bs = 0;        // G == 2: largest block size in the batch
    bool no_generic = false;    // CLX_OPT_NO_GENERIC: no generic-kernel launch after a fast path
    bool no_wide = false;       // CLX_OPT_NO_WIDE: G == 2 without its i64 second chance
};
// clx_fused.cu: `which` bit 0 = index pass, bit 1 = decode pass (both in the product; single ones in measurement builds)
size_t seq_scratch_bytes(const CoopPlan& plan, uint32_t n_frames);
cudaError_t launch_seq(const uint8_t* d_bytes, uint64_t buf_bytes, const clx_frame_desc* d_descs, uint32_t n_frames,
                       int32_t* d_out, clx_frame_result* d_results, int* d_need_generic, void* d_params,
                       const CoopPlan& plan, cudaStream_t stream, int which, uint32_t mode = CLX_OUT_PLANAR_I32);
bool coop_plan(uint32_t max_frame_elems, uint32_t max_channels, uint32_t n_frames, int sm_count, size_t smem_budget,
               CoopPlan* plan);
// Bytes of per-subframe parameter scratch the fast path needs for `n_frames` frames.
size_t coop_params_bytes(const CoopPlan& plan, uint32_t n_frames);
// `mode` (G == 2 only): the output mode of the decode pass, see FusedOut.
cudaError_t launch_coop(const uint8_t* d_bytes, uint64_t buf_bytes, const clx_frame_desc* d_descs, uint32_t n_frames,
                        int32_t* d_out, clx_frame_result* d_results, int* d_need_generic, void* d_params,
                        const CoopPlan& plan, cudaStream_t stream, uint32_t mode = CLX_OUT_PLANAR_I32);
// Interleaved output written by the decode pass of G == 2 itself (a device-resident batch in mode
// CLX_OUT_INTERLEAVED_I32 / _I16): the fast kernels write `d_dst` directly.  The generic kernel stays planar and
// writes d_out; `d_mark` (one byte per frame) records which frames it takes over, and only those are converted
// into d_dst after it, by a pass that exits at once when the fast path declined nothing.
struct FusedOut {
    uint32_t mode;
    void* d_dst;
    uint8_t* d_mark;
    uint32_t max_frame_elems;  // largest n_channels * block_size of the batch
};
// Decodes `n_frames` frames described by d_descs from d_bytes (256-byte aligned; buf_bytes = allocated
// size, a multiple of 64 with at least 128 bytes of slack after the last frame) into
// d_out / d_results on `stream`.  d_need_hi is a 4-byte device scratch word.
// d_flags: two device ints of scratch.  `plan` (may have G == 0) selects the cooperative fast path.
cudaError_t launch_decode(const uint8_t* d_bytes, uint64_t buf_bytes, const clx_frame_desc* d_descs,
                          uint32_t n_frames, int32_t* d_out, clx_frame_result* d_results, int* d_flags,
                          void* d_params, const CoopPlan& plan, cudaStream_t stream, uint64_t* launches,
                          const FusedOut* fused = nullptr);
// clx_crc.cu: frame CRC-16 of every frame that decoded (over the length the decode found), on the device
cudaError_t crc16_init();  // once per context, on its device
cudaError_t launch_crc16(const uint8_t* d_bytes, const clx_frame_desc* d_descs, uint32_t n_frames, clx_frame_result* d_results,
                         cudaStream_t stream);
// clx_output.cu: planar i32 -> interleaved little-endian samples (CLX_OUT_* modes), frame by frame
uint32_t output_elem_size(uint32_t mode);
// `sel` (optional): only frames f with sel[f] != 0; `gate` (optional): nothing at all while *gate == 0.
cudaError_t launch_interleave(const clx_frame_desc* d_descs, uint32_t n_frames, uint32_t max_frame_elems, const int32_t* d_planar,
                              void* d_dst, uint32_t mode, cudaStream_t stream, const uint8_t* sel = nullptr,
                              const int* gate = nullptr);
// mark[f] = (results[f].status == status) for every frame, unless *gate == 0 (then nothing is written).
cudaError_t launch_mark_status(const clx_frame_result* d_results, uint32_t n_frames, int32_t status, uint8_t* d_mark,
                               const int* gate, cudaStream_t stream);
#ifdef CLX_EXPERIMENT
extern int g_exp_which;  // measurement builds only: bit 0 = index pass, bit 1 = decode pass of G == 2
extern int g_exp_dyn_smem;
#endif

}  // namespace clx
#endif
