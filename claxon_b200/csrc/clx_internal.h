// clx_internal.h — shared between the kernels (clx_decode.cu) and the C ABI (clx_api.cu).
#ifndef CLX_INTERNAL_H
#define CLX_INTERNAL_H
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
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
// How a set of frames is decoded (make_plan in clx_api.cu).
enum class Path {
    Generic,       // the generic lane-per-frame kernel alone (clx_decode.cu)
    WarpPerFrame,  // entropy decode + prediction (clx_coop.cu), then the generic kernel for what they declined
    LanePerFrame,  // index pass + lane-per-subframe decode pass (clx_fused.cu), then the generic kernel likewise
};
struct Plan {
    Path path = Path::Generic;
    uint32_t channels = 0;         // fast paths: channel slots per frame (power of two >= max channels of the set)
    uint32_t max_frame_elems = 0;  // largest n_channels * block_size of the set
    bool no_generic = false;       // CLX_OPT_NO_GENERIC: no generic-kernel launch after a fast path
    bool no_wide = false;          // CLX_OPT_NO_WIDE: LanePerFrame without its i64 second chance
};
// Bytes of per-subframe parameter scratch the plan's path needs for `n_frames` frames.
size_t coop_params_bytes(const Plan& plan, uint32_t n_frames);
size_t seq_scratch_bytes(const Plan& plan, uint32_t n_frames);

// The device buffers of one decode.  `bytes`: 256-byte aligned, buf_bytes = allocated size, a multiple of 64 with at
// least 128 bytes of slack after the last frame.  `flags`: four device ints of scratch.  `out`: planar i32 (the
// output in mode CLX_OUT_PLANAR_I32, else the generic kernel's scratch); `conv`: the output of an interleaved or
// channels mode.  `mark` (one byte per frame, optional): given, a LanePerFrame decode to interleaved I32 / I16 or to a
// channels mode writes `conv` itself; `mark` then records which frames the generic kernel takes over, and only those
// are converted after it.  Channels modes only: `cols`, per frame in the order of `descs` (whose out_offset is then the
// frame's place in the planar scratch `out`), the element of `conv` where the frame's window starts on its first row
// (row base * stride + column); `stride`, the row length of `conv`; `wins`, the frame's window, first | count << 16:
// samples [first, first + count) of each channel are stored, no other element is written.
struct DecodeBuffers {
    const uint8_t* bytes;
    uint64_t buf_bytes;
    const clx_frame_desc* descs;
    uint32_t n_frames;
    int32_t* out;
    clx_frame_result* results;
    int* flags;
    void* params;
    uint32_t mode;
    void* conv;
    uint8_t* mark;
    const uint64_t* cols;
    uint64_t stride;
    const uint32_t* wins;
};
// The whole launch sequence of one decode on `stream`: the plan's kernels, the device CRC-16 when `crc`, the
// conversion to an interleaved mode.  Every kernel launched adds one to *launches.
cudaError_t launch_decode(const DecodeBuffers& b, const Plan& plan, bool crc, cudaStream_t stream, uint64_t* launches);

// Launchers of the fast paths' kernels, next to them.  `need_generic` / `need_wide`: device flag words.
cudaError_t launch_warp_per_frame(const uint8_t* d_bytes, uint64_t buf_bytes, const clx_frame_desc* d_descs, uint32_t n_frames,
                                  int32_t* d_out, clx_frame_result* d_results, int* d_need_generic, void* d_params,
                                  const Plan& plan, cudaStream_t stream, uint64_t* launches);
// `mode`: the output mode the decode pass writes (planar, or interleaved I32 / I16 or channels I32 / F32 into `d_out`;
// `d_cols` / `stride` / `d_wins` as in DecodeBuffers).
cudaError_t launch_seq(const uint8_t* d_bytes, uint64_t buf_bytes, const clx_frame_desc* d_descs, uint32_t n_frames,
                       int32_t* d_out, clx_frame_result* d_results, int* d_need_generic, int* d_need_wide, void* d_params,
                       const Plan& plan, uint32_t mode, const uint64_t* d_cols, uint64_t stride, const uint32_t* d_wins,
                       cudaStream_t stream, uint64_t* launches);
// clx_crc.cu: frame CRC-16 of every frame that decoded (over the length the decode found), on the device
cudaError_t crc16_init();  // once per context, on its device
cudaError_t launch_crc16(const uint8_t* d_bytes, const clx_frame_desc* d_descs, uint32_t n_frames, clx_frame_result* d_results,
                         cudaStream_t stream, uint64_t* launches);
// clx_output.cu: planar i32 -> interleaved little-endian samples (CLX_OUT_* modes), frame by frame
uint32_t output_elem_size(uint32_t mode);
// `sel` (optional): only frames f with sel[f] != 0; `gate` (optional): nothing at all while *gate == 0.
cudaError_t launch_interleave(const clx_frame_desc* d_descs, uint32_t n_frames, uint32_t max_frame_elems, const int32_t* d_planar,
                              void* d_dst, uint32_t mode, cudaStream_t stream, uint64_t* launches, const uint8_t* sel = nullptr,
                              const int* gate = nullptr);
// planar i32 -> channels-first i32 / f32 (CLX_OUT_CHANNELS_*): samples [first, first + count) of channel c of frame f
// (d_wins[f] = first | count << 16) at d_dst + c * stride + d_cols[f].  `sel` / `gate` as for launch_interleave.
cudaError_t launch_channels(const clx_frame_desc* d_descs, uint32_t n_frames, uint32_t max_frame_elems, const int32_t* d_planar,
                            void* d_dst, const uint64_t* d_cols, uint64_t stride, const uint32_t* d_wins, uint32_t mode,
                            cudaStream_t stream,
                            uint64_t* launches, const uint8_t* sel = nullptr, const int* gate = nullptr);
// mark[f] = (results[f].status == status) for every frame, unless *gate == 0 (then nothing is written).
cudaError_t launch_mark_status(const clx_frame_result* d_results, uint32_t n_frames, int32_t status, uint8_t* d_mark,
                               const int* gate, cudaStream_t stream, uint64_t* launches);
// clx_crops.cu: crop and packed batches.  A corpus on the device: its descriptors (descs[n_frames] is the filler frame),
// each frame's first sample within its file, each file's frame range [file_frames[i], file_frames[i + 1]), length,
// channel count and trailing-bytes verdict.  A corpus in host memory (CLX_CORPUS_HOST) also gives the device address of
// its mapped pinned bytes and the size of the batch's staging buffer: each call gathers the excerpts' spans of frames
// into it, the filler frame follows at `staging`, and the descriptors point there.  Both are 0 for a device corpus.
struct CropCorpus {
    const clx_frame_desc* descs;
    const int64_t* starts;
    const uint32_t* file_frames;
    const int64_t* file_len;
    const uint32_t* file_ch;
    const int32_t* file_tail;
    uint32_t n_files, n_frames;
    const uint8_t* host_bytes;
    uint64_t staging;
};
// Per excerpt, what the planner found (device memory, written every decode).
struct ExcerptPlan {
    int64_t lo;       // first sample of the excerpt
    uint32_t count;   // frames overlapping it
    uint32_t first;   // corpus index of the first of them
    uint32_t file;
    uint32_t ch;      // rows the excerpt covers (0: an invalid request)
};
// The excerpts of a crop or packed batch (and the requests, lengths and layout of a resampled one).  A crop batch is
// a packed batch whose excerpts each own a row group: where an excerpt's output starts, whether it fits and what is
// zeroed around it is the layout's (CropLayout, PackedLayout in clx_scan.cuh), everything else is shared.  Over a host
// corpus the staging buffer holds each excerpt's span at stage[b], the scan of span bytes + 15 moved up to the span
// start's residue mod 16.
struct ExcerptBuffers {
    const clx_crop_request* crop_requests;      // crop batches: n requests, length L
    const clx_packed_request* packed_requests;  // packed batches: n requests ...
    const uint32_t* count;                      // ... of which this call uses the first *count (device, by the caller)
    int32_t* status;
    int64_t* lengths;
    unsigned long long* error;
    ExcerptPlan* plan;
    uint32_t* scan;   // n + 1: exclusive scan of the slots, then the total
    int64_t* starts;  // packed batches: each excerpt's first column
    uint64_t* stage;  // host corpus: where each excerpt's span starts in the staging buffer
    uint32_t* chunks; // n + 1: exclusive scan of each span's gather chunks, then the total
    uint64_t* end;    // packed batches: [0] this call's end column, [1] the previous call's
    uint32_t n, C, n_slots;
    uint32_t slot_elems;
    uint64_t L;       // the row length: num_frames of a crop batch, the stride of a packed one (trash columns included)
    uint64_t T;       // packed batches: max_samples, the columns users see
};
// Kernels take it by value.  Above 128 bytes nvcc reads such a parameter through a pointer, which took the gather's
// per-excerpt values off the uniform datapath (40 registers instead of 32).
static_assert(sizeof(ExcerptBuffers) <= 128, "ExcerptBuffers is a kernel parameter of at most 128 bytes");
struct CropLayout;
struct PackedLayout;
// Filler frame: 1 channel, 16 bits, block size 192, CONSTANT 0.  Writes it if cap suffices; returns its length.
size_t filler_frame(uint8_t* out, size_t cap);
// clx_api.cu, for corpus images (clx_corpus_image.cpp): the size of a frame-bytes buffer of `nbytes` bytes (whole
// 64-byte chunks + 128 bytes of look-ahead); the per-frame checks of clx_corpus_create_ex (byte range and the shapes the
// kernels decode); the trailing-bytes verdict of a file whose last frame `d` has an unconfirmed end.
size_t padded_bytes(size_t nbytes);
bool corpus_frames_ok(const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames);
int tail_verdict(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, clx_frame_desc d, int32_t* verdict);
// clx_corpus_image.cpp: what clx_corpus_attach takes from an image that clx_corpus_image_check accepted, copied out of
// it.  descs: n_frames + 1, the filler frame last, byte_offset into the bytes region; file_frames: n_files + 1.
struct ImageIndex {
    uint64_t bytes_offset = 0, bytes_size = 0, nbytes = 0;
    std::vector<clx_frame_desc> descs;
    std::vector<uint32_t> file_frames;
    std::vector<int32_t> tail;
};
// CLX_OK with `ix` filled, or CLX_ERR_INVALID_ARGUMENT (clx_corpus_image_check's verdict).
int read_image(const void* image, size_t image_bytes, ImageIndex* ix);
// The launch sequence of a crop (Layout = CropLayout) or packed batch (PackedLayout): planner (count, scan, the gather
// of a host corpus, emit, zero-fill), launch_decode over every slot, status pass.  `db`: the batch's buffers;
// db.descs / db.cols / db.wins are written by the planner, and over a host corpus db.bytes is the staging buffer the
// gather writes.
template <class Layout>
cudaError_t launch_excerpts(const CropCorpus& cc, const ExcerptBuffers& eb, const DecodeBuffers& db, const Plan& plan,
                            bool crc, cudaStream_t stream, uint64_t* launches);

// clx_resample.cu: resampled crop batches (clx_batch_create_resampled_crops), a packed batch of each crop's source span
// between two kernels.  One polyphase table per distinct source rate r != R: with g = gcd(r, R), o = r / g, n = R / g,
// output blk * n + ph is sum_i coef[i * n + ph] * x[blk * o + k0[ph] + i]; taps 0 marks r == R (copied).
struct ResampleRate {
    uint32_t o, n, w, taps;
    uint64_t coef;  // the table's first coefficient in ResampleBuffers::coefs
    uint64_t k0;    // its first k0 in ResampleBuffers::k0 (n of them, each in [-w, w + o - taps])
};
// Per crop, what resample_map_kernel found (device memory, written every decode).
struct ResamplePlan {
    int64_t offset;            // first output sample, at rate R
    int64_t src_lo, src_len;   // the source span decoded for it: samples [src_lo, src_lo + src_len) of its file
    uint32_t rate;             // its file's ResampleRate
    uint32_t ch;               // rows the crop covers (0: an invalid request)
};
struct ResampleBuffers {
    int64_t* lengths;               // at rate R
    ResamplePlan* plan;
    const uint32_t* file_rate;      // per file, its ResampleRate
    const ResampleRate* rates;
    const float* coefs;
    const int32_t* k0;
    clx_packed_request* excerpts;   // the inner packed batch's requests and count, written by the map kernel
    uint32_t* count;
    const int64_t* starts;          // ... its column starts
    const float* src;               // ... and output, rows of src_stride
    uint64_t src_stride;
    float* out;                     // [n_crops * C, L]
    uint32_t n_crops, C, tile;      // tile: outputs per CTA of resample_kernel
    uint64_t L;
};
// The host side of clx_batch_create_resampled_crops: the tables of the distinct rates of file_rates towards target, and
// the longest source span of a crop (clx_resample_source_bound over those rates).  false for a rate of 0 or above
// CLX_MAX_SAMPLE_RATE, or more than 2^24 coefficients in all.
struct ResampleTables {
    std::vector<ResampleRate> rates;
    std::vector<uint32_t> file_rate;
    std::vector<float> coefs;
    std::vector<int32_t> k0;
    uint64_t bound = 0;
    uint32_t tile = 0;
};
bool resample_tables(const uint32_t* file_rates, size_t n_files, uint32_t target, size_t num_frames, ResampleTables* t);
// The map kernel before the inner packed batch's launch sequence, of a resampled crop (Layout = CropLayout) or packed
// batch (PackedLayout): `eb` holds the batch's own requests at rate R (and count, target column starts and T of a
// packed one).  Then the filter kernel of a crop batch.
template <class Layout>
cudaError_t launch_resample_map(const CropCorpus& cc, const ResampleBuffers& rs, const ExcerptBuffers& eb,
                                cudaStream_t stream, uint64_t* launches);
cudaError_t launch_resample(const ResampleBuffers& rs, cudaStream_t stream, uint64_t* launches);
// Resampled packed batches (clx_batch_create_resampled_packed) keep the same ResampleBuffers, with n_crops =
// max_excerpts, L = the output's row stride and lengths at rate R.  The inner packed batch has resample_packed_bound
// columns (clx_resample_packed_source_bound over t's rates).
size_t resample_packed_bound(const ResampleTables& t, size_t max_excerpts, size_t max_samples);
cudaError_t launch_resample_packed(const ResampleBuffers& rs, const ExcerptBuffers& eb, cudaStream_t stream,
                                   uint64_t* launches);

// clx_mel.cu: mel crop batches (clx_batch_create_mel_crops), one kernel after an inner crop or resampled crop batch
// (two with a CLX_MEL_NORM_* flag).
// Mel m sums weights[w + i] * |X[lo + i]|^2 for i < n: the non-zero span of its filterbank column.
struct MelBand {
    uint32_t lo, n, w;
};
struct MelBuffers {
    const float* src;       // the inner batch's [rows, L] output
    float* out;             // [rows, n_mels, F]
    const float* tw;        // n_fft complex: exp(-2 pi i k / n_fft)
    const float* window;    // n_fft: the window at (n_fft - win_length) / 2, zeros around it
    const MelBand* bands;   // n_mels
    const float* weights;
    uint64_t L, F;
    uint32_t rows, tiles;   // CTAs: rows * tiles
    uint32_t n_fft, hop, n_mels, tile;  // tile: frames per CTA
    uint32_t flags;         // CLX_MEL_*
    float log_floor, log_of_floor;  // ln(log_floor), taken in float64
};
// The host side of clx_batch_create_mel_crops and _mel_packed: the checks of the header's refusals that depend neither
// on the inner batch nor on a row length, and the tables.  false for a refusal.  mel_params_ok: those checks of the
// parameters alone (params not NULL included).
struct MelTables {
    std::vector<float> tw, window, weights;
    std::vector<MelBand> bands;
    uint32_t tile = 0;
    size_t smem = 0;
};
bool mel_params_ok(const clx_mel_params* p);
bool mel_tables(const clx_mel_params* p, const float* window, const float* fbank, MelTables* t);
cudaError_t mel_init();  // the mel kernels' shared memory limit, on the current device, before a graph captures them
// mel_norm_kernel's view of a mel batch with CLX_MEL_NORM_* in flags (flags 0: no normalisation, no launch).  Crops:
// segment (crop b, row c, mel m) is out[((b C + c) n_mels + m) F ...], its valid frames 1 + lengths[b] / hop.  Packed
// (count set): out[(c n_mels + m) F + starts[b] ...], frames[b] of them, for b < min(*count, n).
struct MelNorm {
    float* out;
    const int64_t* lengths;  // crops: each crop's length in samples
    const uint32_t* count;   // packed: the call's excerpt count; NULL for crops
    const int64_t* starts;   // packed: frame starts and counts (the planner's)
    const int64_t* frames;
    uint64_t F;              // the row pitch: frames of a crop row, T_f of a packed batch
    uint32_t n, C, n_mels, hop;  // n: crops, or max_excerpts
    uint32_t flags;          // CLX_MEL_NORM_PER_FEATURE or CLX_MEL_NORM_WHISPER, or 0
};
cudaError_t launch_mel(const MelBuffers& mb, const MelNorm& mn, size_t smem, cudaStream_t stream, uint64_t* launches);
// Mel packed batches (clx_batch_create_mel_packed) keep a MelBuffers with src = the inner packed batch's [C, L] output
// (L its row stride), rows = C, F = the frame columns T_f (the features' row pitch), and this: the inner batch's count,
// lengths in samples and sample starts, and the batch's own frame starts and frame counts, written by the planner.
struct MelPacked {
    const uint32_t* count;
    const int64_t* lengths;
    const int64_t* src_starts;
    int64_t* starts;
    int64_t* frames;
    uint32_t n;  // max_excerpts
};
// clx_mel_packed_frames_bound of valid parameters: SIZE_MAX if it overflows.
size_t mel_packed_frames(const clx_mel_params* p, size_t max_excerpts, size_t max_samples);
// The planner (frame counts and starts), mel_packed_kernel and, with mn.flags, mel_norm_kernel, after the inner batch's
// launch sequence.
cudaError_t launch_mel_packed(const MelBuffers& mb, const MelPacked& mp, const MelNorm& mn, size_t smem,
                              cudaStream_t stream, uint64_t* launches);
#ifdef CLX_EXPERIMENT
extern int g_exp_which;  // measurement builds only: bit 0 = index pass, bit 1 = decode pass of LanePerFrame
extern int g_exp_dyn_smem;
#endif

}  // namespace clx
#endif
