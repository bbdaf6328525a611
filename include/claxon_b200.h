/* claxon_b200.h — C ABI of the H100-native batched FLAC frame decoder.
 *
 * This is the drop-in boundary for the per-frame decode path of ruuda/claxon
 * v0.4.3.  claxon has no FFI of its own; its boundary is the Rust API
 *   FrameReader::read_next_or_eof(&mut self, Vec<i32>) -> Result<Option<Block>>
 *                                                     (reference src/frame.rs:667)
 *   FlacReader::{new, streaminfo, blocks, samples}    (src/lib.rs:217-435)
 *   Block::{time, len, duration, channels, channel, sample, into_buffer}
 *                                                     (src/frame.rs:402-529)
 * A Rust `extern "C"` shim (INTEGRATION.md) binds exactly the entry points below:
 * the host parses frame headers (clx_parse_frame_header == src/frame.rs:131-316),
 * ships raw frame bitstreams to the device, and everything below the header parse
 * and above the CRC-16 footer check — subframe::decode (src/subframe.rs:184-228),
 * decode_residual (:236-380), predict_fixed (:417-474), predict_lpc_* (:524-614),
 * decode_{left,right,mid}_side (src/frame.rs:319-389) — runs in sm_90a kernels.
 *
 * Plain pointers and sizes only; no torch / C++ types cross this boundary.
 * There is NO CPU fallback: if no CUDA device is usable the create call fails
 * with CLX_ERR_NO_DEVICE.
 */
#ifndef CLAXON_B200_H
#define CLAXON_B200_H

#include <stddef.h>
#include <stdint.h>
#include "clx_status.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CLX_ABI_VERSION 1

/* ------------------------------------------------------------------------- */
/* Frame descriptor: the parsed frame header + where the frame's bytes are.   */
/* Mirrors claxon's private FrameHeader (src/frame.rs:41-48).                 */
/* ------------------------------------------------------------------------- */
typedef struct clx_frame_desc {
    uint64_t byte_offset;        /* offset of the frame's first sync byte in the byte buffer */
    uint32_t byte_len;           /* bytes AVAILABLE to this frame from byte_offset: the exact frame
                                    length (sync..CRC-16) when known, else an upper bound (e.g. to
                                    the end of the stream).  Reads past it are UnexpectedEof. */
    uint16_t header_len;         /* frame header bytes incl. the CRC-8 */
    uint16_t block_size;         /* 1..65535 inter-channel samples */
    uint8_t n_channels;          /* 1..8 */
    uint8_t channel_assignment;  /* raw 4-bit code: 0..7 independent(n+1), 8 L/S, 9 R/S, 10 M/S */
    uint8_t bits_per_sample;     /* 8/12/16/20/24; 0 = not in the header (-> Unsupported) */
    uint8_t flags;               /* CLX_FRAME_* */
    uint32_t sample_rate;        /* Hz, 0 = "from streaminfo"; not used by the decode */
    uint64_t number;             /* coded frame / sample number */
    uint64_t out_offset;         /* element (i32) offset of this frame's samples in the output;
                                    multiple of 4 recommended (vectorised stores).  Elements of
                                    `out` that lie between the first and the last frame of a call but
                                    belong to no frame (alignment gaps) are unspecified afterwards. */
} clx_frame_desc;

#define CLX_FRAME_VARIABLE_BLOCKING 1u /* `number` is a sample number, else a frame number */
#define CLX_FRAME_CRC16_VERIFIED 2u    /* set by clx_demux_frames: CRC-16 of the first byte_len-2 bytes
                                          already matched the footer (saves the host a second pass) */

/* Per-frame outcome. */
typedef struct clx_frame_result {
    int32_t status;      /* clx_status; CLX_OK when the frame decoded and its CRC-16 matched */
    uint32_t consumed;   /* bytes from the sync code through the CRC-16 (valid when status is
                            CLX_OK or CLX_ERR_FRAME_CRC_MISMATCH) */
} clx_frame_result;

/* STREAMINFO (src/metadata.rs:29-54). 0 = unknown for frame sizes / samples. */
typedef struct clx_streaminfo {
    uint32_t min_block_size, max_block_size;
    uint32_t min_frame_size, max_frame_size;
    uint32_t sample_rate, channels, bits_per_sample;
    uint64_t samples;
    uint8_t md5sum[16];
} clx_streaminfo;

typedef struct clx_options {
    int32_t device;        /* CUDA device ordinal */
    uint32_t flags;        /* CLX_OPT_* */
    uint32_t n_streams;    /* internal CUDA streams for host<->device pipelining (0 = default 2) */
    uint32_t host_threads; /* host threads for the CRC-16 pass (0 = default: min(32, hardware threads));
                              give each rank its share when several ranks run on one host */
} clx_options;
#define CLX_OPT_NO_VERIFY_CRC 1u /* mimic claxon's cfg(fuzzing): skip CRC-8/CRC-16 checks */
#define CLX_OPT_GENERIC_KERNEL_ONLY 2u /* testing: bypass the fast path */
#define CLX_OPT_WARP_PER_FRAME 4u      /* the warp-per-frame fast path everywhere (default: only for small synchronous calls) */
#define CLX_OPT_LANE_PER_FRAME 8u      /* the lane-per-frame fast path everywhere, also for small synchronous calls */
/* Testing: a fast path's verdicts are left as they are.  NO_GENERIC: the generic kernel does not re-decode the frames
 * a fast path declined (a call without a fast path still runs it); such a frame comes back with status -2.
 * NO_WIDE: the lane-per-frame path skips its i64 second chance; a frame that needed it comes back with status -3.
 * Neither status ever reaches the caller without these options. */
#define CLX_OPT_NO_GENERIC 16u
#define CLX_OPT_NO_WIDE 32u

typedef struct clx_ctx clx_ctx;     /* one per host thread / GPU; owns device scratch */
typedef struct clx_batch clx_batch; /* a device-resident batch (bytes + descriptors + output) */

/* ------------------------------------------------------------------------- */
/* status helpers                                                             */
/* ------------------------------------------------------------------------- */
const char* clx_status_str(int status);  /* claxon's verbatim error string */
int clx_status_kind(int status);         /* clx_error_kind */
uint32_t clx_abi_version(void);

/* ------------------------------------------------------------------------- */
/* host-side parsing (no GPU needed)                                          */
/* ------------------------------------------------------------------------- */

/* read_frame_header_or_eof (src/frame.rs:131-316) on p[0..n).  Fills every field of
 * `d` except byte_offset/byte_len/out_offset.  CLX_EOF when fewer than 2 bytes remain. */
int clx_parse_frame_header(const uint8_t* p, size_t n, clx_frame_desc* d, uint32_t flags);

/* FlacReader::new (src/lib.rs:217-307, default options): checks 'fLaC', walks the
 * metadata blocks, returns STREAMINFO and the offset of the first frame. */
int clx_open_stream(const uint8_t* p, size_t n, clx_streaminfo* si, uint64_t* first_frame);
/* FlacReader::new_ext with FlacReaderOptions (src/lib.rs:123-170, :230-307).  CLX_OPEN_METADATA_ONLY: stop
 * as soon as every desired block has been read; *first_frame is then 0 and the stream cannot be decoded
 * (claxon panics in blocks()/samples()).  CLX_OPEN_NO_VORBIS_COMMENT == read_vorbis_comment: false.
 * *vc_offset / *vc_length locate the body of the (validated) VORBIS_COMMENT block, 0 / 0 when there is
 * none or it was not asked for: little-endian u32 vendor length, vendor string, u32 comment count, then
 * per comment a u32 length and "NAME=value" in UTF-8 (what FlacReader::vendor/tags/get_tag expose,
 * src/lib.rs:318-360, src/metadata.rs:134-211); zero-length comments are to be skipped. */
#define CLX_OPEN_METADATA_ONLY 1u
#define CLX_OPEN_NO_VORBIS_COMMENT 2u
int clx_open_stream_ex(const uint8_t* p, size_t n, uint32_t open_flags, clx_streaminfo* si, uint64_t* first_frame,
                       uint64_t* vc_offset, uint32_t* vc_length);

/* Frame demultiplexer: finds frame boundaries in bytes[start..n) without decoding:
 * sync code + header parse + CRC-8, then the first later sync position at which the
 * CRC-16 over the candidate span matches (or the end of the stream).  Writes up to
 * `max_frames` descriptors with exact byte_len and out_offset laid out back to back
 * (each frame aligned to 4 elements).  Stops at the first position that is not a
 * valid frame start and reports that header's status in *stop_status (CLX_EOF at a
 * clean end).  Returns the number of descriptors written. */
size_t clx_demux_frames(const uint8_t* bytes, size_t n, uint64_t start, clx_frame_desc* descs,
                        size_t max_frames, uint64_t* next_offset, uint64_t* total_out_elems,
                        int* stop_status, uint32_t flags);

/* The same on `n_threads` host threads (0 = one per hardware thread): the byte range is cut into equal parts, every
 * worker finds the frames that START in its part — a start counts once its header parses (sync code, field codes,
 * CRC-8) and a CRC-16-confirmed end lies within the size that header allows — and the parts are stitched in order,
 * a part being accepted only if the chain before it ends exactly where it begins.  Descriptor for descriptor the
 * result of clx_demux_frames; the scan (dominated by the CRC-16 of every byte) runs at n_threads times its rate. */
size_t clx_demux_frames_mt(const uint8_t* bytes, size_t n, uint64_t start, clx_frame_desc* descs,
                           size_t max_frames, uint64_t* next_offset, uint64_t* total_out_elems,
                           int* stop_status, uint32_t flags, uint32_t n_threads);

/* Container feeds (SURVEY.md §8 f4): a wrapper that stores one FLAC frame per packet / sample hands over
 * the frame boundaries, so no search (clx_demux_frames) is needed.  What the reference leaves to the `ogg`
 * and `mp4parse` crates in examples/decode_ogg.rs:26-125 and examples/decode_mp4.rs:26-167.
 *
 * clx_ogg_frames: an in-memory Ogg file with the FLAC mapping (first packet: 0x7F "FLAC" version, number of
 * header packets, "fLaC", STREAMINFO; then the header packets; then one frame per packet; empty packets
 * skipped; page CRCs verified unless CLX_OPT_NO_VERIFY_CRC).  Packets may span pages, so the frames are
 * copied back to back into `frames_out` (capacity frames_cap; the file's size always suffices) and the
 * descriptors index THAT buffer; byte_len is exact.
 * clx_mp4_frames: an in-memory MP4 / ISO BMFF file; the first track with a 'fLaC' sample entry.  STREAMINFO
 * comes from its dfLa box, frame extents from stsz + stsc + stco/co64; samples are contiguous in the file, so
 * the descriptors index the file's own bytes.
 * Both fill out_offset back to back (4-element aligned) and return CLX_ERR_CONTAINER for a malformed wrapper,
 * a frame-header status if a packet / sample is not a frame, CLX_ERR_INVALID_ARGUMENT if max_frames or
 * frames_cap is too small. */
int clx_ogg_frames(const uint8_t* ogg, size_t n, clx_streaminfo* si, uint8_t* frames_out, size_t frames_cap,
                   clx_frame_desc* descs, size_t max_frames, size_t* n_frames, size_t* frames_bytes,
                   uint64_t* total_out_elems, uint32_t flags);
int clx_mp4_frames(const uint8_t* mp4, size_t n, clx_streaminfo* si, clx_frame_desc* descs, size_t max_frames,
                   size_t* n_frames, uint64_t* total_out_elems, uint32_t flags);

uint8_t clx_crc8(const uint8_t* p, size_t n);   /* src/crc.rs: poly 0x07, init 0 */
uint16_t clx_crc16(const uint8_t* p, size_t n); /* src/crc.rs: poly 0x8005, init 0 */

/* ------------------------------------------------------------------------- */
/* device path                                                                */
/* ------------------------------------------------------------------------- */
int clx_ctx_create(const clx_options* opts, clx_ctx** out);
void clx_ctx_destroy(clx_ctx* ctx);
const char* clx_ctx_last_error(const clx_ctx* ctx); /* CUDA error text for CLX_ERR_CUDA */

/* The per-frame decode path, end to end with HOST buffers (the call a binding makes):
 * copies the frame bytes to the device, runs the decode kernels, copies the planar
 * i32 PCM (Block layout: buffer[ch*block_size + i], src/frame.rs:477-481) back into
 * `out` at descs[i].out_offset, and fills results[i].  The frame CRC-16 is verified
 * (unless CLX_OPT_NO_VERIFY_CRC) after the subframes, so subframe errors pre-empt
 * "frame CRC mismatch" exactly as in src/frame.rs:752-763.  A failed frame never
 * aborts the batch; its output region is fully overwritten (never stale). */
int clx_decode_frames(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                      size_t n_frames, int32_t* out, size_t out_elems, clx_frame_result* results);

/* Output stage (SURVEY.md §8 f2): the same call with the samples delivered INTERLEAVED — for each
 * inter-channel sample every channel in turn, the order FlacSamples yields them in (src/lib.rs:473-519)
 * — as little-endian integers of 2, 3 or 4 bytes: what a WAV writer stores (examples/decode.rs:48-62)
 * and what the STREAMINFO MD5 is defined over (src/metadata.rs:52-53).  The conversion runs on the
 * device, so 16-bit audio crosses PCIe as 2 bytes per sample.  `out_elems` and descs[i].out_offset
 * count SAMPLES (elements of 2 / 3 / 4 bytes); a frame occupies n_channels * block_size of them as in
 * the planar layout.  CLX_OUT_INTERLEAVED_I16 / _I24 require every frame's bits_per_sample to be at
 * most 16 / 24 (else CLX_ERR_INVALID_ARGUMENT); a sample that nevertheless does not fit (only an invalid
 * stream has them) is truncated to the element size like `sample as i16` in examples/decode.rs:52.
 * CLX_OUT_PLANAR_I32 is clx_decode_frames. */
#define CLX_OUT_PLANAR_I32 0u
#define CLX_OUT_INTERLEAVED_I32 1u
#define CLX_OUT_INTERLEAVED_I16 2u
#define CLX_OUT_INTERLEAVED_I24 3u
int clx_decode_frames_to(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                         size_t n_frames, void* out, size_t out_elems, clx_frame_result* results, uint32_t mode);

/* Device-resident variant: upload once, decode many times (kernel-only timing), read back. */
int clx_batch_create(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                     size_t n_frames, size_t out_elems, clx_batch** out);
/* The same with `bytes` in DEVICE memory of the context's GPU (CLX_BATCH_BYTES_ON_DEVICE): e.g. a shard that
 * arrived over NVLink by the one NCCL scatter (claxon_b200/shard.py).  Nothing of it ever passes through the host:
 * the frame CRC-16 is then checked on the device as part of every decode. */
#define CLX_BATCH_BYTES_ON_DEVICE 1u
int clx_batch_create_ex(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                        size_t n_frames, size_t out_elems, uint32_t batch_flags, clx_batch** out);
/* Output modes for device-resident batches: the same batch with its samples kept in one of the CLX_OUT_* forms of
 * clx_decode_frames_to, so that a consumer that stays on the device (clx_batch_device_out) gets what a WAV writer or
 * the STREAMINFO MD5 uses without a conversion pass of its own.  `out_elems` and descs[i].out_offset count SAMPLES
 * (elements of 2 / 3 / 4 bytes) as in clx_decode_frames_to, and the same rules hold: CLX_OUT_INTERLEAVED_I16 / _I24
 * require every frame's bits_per_sample to be at most 16 / 24 (else CLX_ERR_INVALID_ARGUMENT, as for a mode above
 * CLX_OUT_INTERLEAVED_I24), a sample that does not fit is truncated like `sample as i16`, and a failed frame's
 * region is fully overwritten.  On the lane-per-frame path the I32 and I16 forms are written by the decode kernel
 * itself; I24, and every other path, convert from planar inside the batch's graph.  clx_batch_create_ex is this call
 * with CLX_OUT_PLANAR_I32. */
int clx_batch_create_to(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                        size_t n_frames, size_t out_elems, uint32_t batch_flags, uint32_t mode, clx_batch** out);
/* Channels-first output for device-resident batches: one [n_channels, channel_stride] buffer of 4-byte elements, the
 * layout PyTorch audio code uses (one row per channel, time along the row).  In these modes descs[i].out_offset is
 * the frame's COLUMN: row c < descs[i].n_channels gets that channel's block_size samples at columns [out_offset,
 * out_offset + block_size), after wasted bits and decorrelation as in the planar layout.  Rows a frame does not have
 * are left alone.  The buffer is zeroed once when the batch is created, so elements that no frame covers read 0 and
 * stay 0.  A failed frame's region is fully overwritten with what the planar layout holds for it, converted.
 * CLX_OUT_CHANNELS_F32 stores (float)s * 2^-(bits_per_sample - 1), bits_per_sample being the frame header's value:
 * the int-to-float conversion rounds to nearest even and the multiply is exact, so every sample of a valid stream of
 * at most 24 bits maps exactly into [-1, 1).
 * CLX_ERR_INVALID_ARGUMENT for: n_channels 0 or above 8, channel_stride 0, n_channels * channel_stride * 4
 * overflowing, a frame with more channels than n_channels or with out_offset + block_size > channel_stride, in F32 a
 * frame with bits_per_sample above 24, a mode other than the two below, and every byte-range condition of the other
 * create calls.  clx_batch_read_to copies min(out_elems, n_channels * channel_stride) elements; clx_batch_read refuses.
 * On the lane-per-frame path the decode kernel writes the rows itself; every other path decodes to a planar scratch
 * buffer and converts inside the batch's graph.  (clx_batch_create_to and clx_decode_frames_to refuse these modes.) */
#define CLX_OUT_CHANNELS_I32 4u /* out[c * channel_stride + t]: sample t of channel c, i32 */
#define CLX_OUT_CHANNELS_F32 5u /* the same as float: (float)s * 2^-(bits_per_sample - 1) */
int clx_batch_create_channels(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                              size_t n_frames, uint32_t n_channels, size_t channel_stride, uint32_t batch_flags,
                              uint32_t mode, clx_batch** out);
/* Channels-first output of sample ranges: each frame stores only a window of its samples, on rows of its own.  This is
 * what a batch of excerpts ("4 s from a random offset of each of B files") needs: the frames that overlap an excerpt
 * are decoded, the first and last of them clipped to it, each excerpt on rows of its own ([B * C, stride] rows).
 * Channel c of frame i goes to row windows[i].row + c; its samples [first, first + count) go to columns
 * [out_offset, out_offset + count) of that row (descs[i].out_offset is the column where sample `first` lands).  No
 * element outside a frame's window is ever written; everything else is as for clx_batch_create_channels (wasted bits
 * and decorrelation applied, the F32 rule, the buffer zeroed once at creation, a failed frame's window overwritten
 * with what the planar layout holds for those samples, converted; clx_batch_read_to, clx_batch_device_out and
 * CLX_BATCH_BYTES_ON_DEVICE as there).  The window {0, 0, block_size} on every frame gives, bit for bit, what
 * clx_batch_create_channels gives.  n_rows has no cap of 8.  Overlapping windows are the caller's business; two
 * descriptors may name the same frame bytes, each is decoded for its own window.
 * CLX_ERR_INVALID_ARGUMENT for: windows NULL with frames, n_rows or row_stride 0, n_rows * row_stride * 4 overflowing,
 * row + n_channels > n_rows, first >= block_size, count 0 or first + count > block_size, out_offset + count >
 * row_stride, reserved != 0, in F32 a frame with bits_per_sample above 24, a mode other than CLX_OUT_CHANNELS_I32 /
 * _F32, and every byte-range condition of the other create calls. */
typedef struct clx_frame_window {
    uint32_t row;      /* channel c of the frame goes to row `row + c` */
    uint32_t first;    /* first sample of the frame that is stored, < block_size */
    uint32_t count;    /* samples stored: 1 .. block_size - first */
    uint32_t reserved; /* 0 */
} clx_frame_window;
int clx_batch_create_windows(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                             const clx_frame_window* windows, size_t n_frames, uint32_t n_rows, size_t row_stride,
                             uint32_t batch_flags, uint32_t mode, clx_batch** out);
/* Device-resident corpora and crop batches: the frames of several FLAC streams uploaded once, and fixed-shape batches of
 * [B, C, L] excerpts of them that plan each call's frames, windows and columns on the device, inside the batch's graph.
 * A call is then: write the requests into clx_batch_crop_requests (device memory), clx_batch_decode; nothing is gathered,
 * uploaded, checksummed or instantiated per call, and the offsets may come from device code.
 *
 * clx_corpus_create: `bytes` (host memory) holds the frames of n_files streams; file i's frames are descs[file_frames[i]
 * .. file_frames[i + 1]) in stream order (file_frames has n_files + 1 entries), byte_offset indexing `bytes`; out_offset
 * is ignored.  Sample t of file i is sample t - start of the frame that holds it, a frame's start being the sum of the
 * block sizes before it in its file.  The bytes and descriptors are uploaded once, with each frame's start and each
 * file's frame range and length.  A file whose last frame lacks CLX_FRAME_CRC16_VERIFIED (its end is unconfirmed) has
 * that frame decoded once here: if it decodes and ends before its byte_len, the frame header status at its end (other
 * than CLX_EOF) is the file's trailing-bytes verdict, reported by every crop that contains that frame.
 * CLX_ERR_INVALID_ARGUMENT for: every descriptor condition of the create calls above, file_frames not monotone or not
 * ending at n_frames, frames of one file with different channel counts, n_frames or n_files of 2^32 - 1 or more.
 * clx_corpus_destroy: CLX_ERR_INVALID_ARGUMENT (and nothing freed) while a crop batch of the corpus is alive.
 *
 * clx_corpus_create_ex: clx_corpus_create with `flags`; 0 is clx_corpus_create.  CLX_CORPUS_HOST keeps the bytes in
 * mapped pinned host memory instead of device memory (host RAM holds them once more, device memory only the frame
 * index: descriptors, starts and the per-file arrays).  Each decode of a crop batch of such a corpus then copies the
 * frames its crops selected over PCIe into a staging buffer of the batch (one more kernel in its graph) and decodes
 * them there, with the same results.  A host corpus also needs each file's frames in byte order: byte_offset and
 * byte_offset + byte_len non-decreasing within a file (as the demuxer gives them).  CLX_ERR_INVALID_ARGUMENT for
 * unknown flag bits and, with CLX_CORPUS_HOST, frames out of byte order; otherwise as clx_corpus_create.
 * clx_corpus_device_bytes: the device memory the corpus holds (its bytes for a device corpus, plus the frame index). */
#define CLX_CORPUS_HOST 1u
typedef struct clx_corpus clx_corpus;
int clx_corpus_create(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                      const uint32_t* file_frames, size_t n_files, clx_corpus** out);
int clx_corpus_create_ex(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                         const uint32_t* file_frames, size_t n_files, uint32_t flags, clx_corpus** out);
int clx_corpus_destroy(clx_ctx* ctx, clx_corpus* corpus);
size_t clx_corpus_device_bytes(const clx_corpus* corpus);
/* The most frames that can overlap num_frames consecutive samples of one file: with m the smallest block size among the
 * frames that are not the last of their file, floor((num_frames - 2) / m) + 2 for num_frames >= 2 and 1 for num_frames
 * 1, but never more than the frames of the largest file (and 1 when no file has two frames).  Host only.  0 for
 * num_frames 0 or a bad file_frames. */
size_t clx_crop_frames_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                             size_t num_frames);
/* The most compressed bytes one crop of num_frames samples can span: with S = clx_crop_frames_bound(num_frames), the
 * largest byte_offset[f + k - 1] + byte_len[f + k - 1] - byte_offset[f] over every frame f, k = min(S, frames of f's
 * file from f on).  Host only, O(n_frames).  0 for num_frames 0 or a bad file_frames. */
size_t clx_crop_bytes_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                            size_t num_frames);
/* A crop batch of n_crops excerpts of num_frames samples each, in mode CLX_OUT_CHANNELS_I32 or _F32.  It is an ordinary
 * clx_batch (clx_batch_decode, _sync, _last_kernel_ms, _read_to, clx_ctx_run_steps, clx_batch_device_out work on it)
 * that shares the corpus's bytes.  Output: [n_crops * C, num_frames] channels-first, C the corpus's largest channel
 * count; crop b is rows [b * C, (b + 1) * C).  Each decode reads request b = {file, reserved, offset}: samples [offset,
 * min(offset + num_frames, length)) of that file go to row b * C + c, columns from 0; every other element of the crop's
 * rows is 0.  A request with file >= n_files, reserved != 0, offset < 0 or offset > length gets status
 * CLX_ERR_INVALID_ARGUMENT, length 0 and zero rows.  Status of a valid crop: the first failed frame in stream order,
 * else the file's trailing-bytes verdict when the crop contains its last frame, else CLX_OK; a failed crop's rows are
 * unspecified.  The frame CRC-16 is checked on the device in every decode (frames the demuxer confirmed are skipped).
 * F32 is refused when ANY frame of the corpus has more than 24 bits, since the batch may be asked for any of them.
 * Memory: (n_crops + 1) * C * num_frames output elements (the C rows after the output take the unused slots) and, per
 * slot, a planar scratch of the corpus's largest frame; slots = n_crops * clx_crop_frames_bound(num_frames).  Over a
 * host corpus (CLX_CORPUS_HOST), also a staging buffer of n_crops spans of clx_crop_bytes_bound(num_frames) + 15 bytes
 * rounded up to 16, plus the filler frame and 128 to 191 bytes of slack; each decode reads every selected crop's span
 * (at most that bound per crop) from host memory over PCIe.
 * CLX_ERR_INVALID_ARGUMENT for: n_crops or num_frames 0, n_crops of 2^30 or more, slots of 2^32 or more, sizes that
 * overflow, a mode other than the two channels modes, F32 with a frame above 24 bits. */
typedef struct clx_crop_request {
    uint32_t file;     /* index of the file in the corpus */
    uint32_t reserved; /* 0 */
    int64_t offset;    /* first sample of the excerpt, 0 .. the file's length */
} clx_crop_request;
int clx_batch_create_crops(clx_ctx* ctx, clx_corpus* corpus, size_t n_crops, size_t num_frames, uint32_t mode,
                           clx_batch** out);
/* Device pointers of a crop batch (NULL for other batches).  requests: n_crops clx_crop_request, written by the caller
 * before clx_batch_decode (zeroed at creation).  status: n_crops int32.  lengths: n_crops int64, min(num_frames,
 * length - offset), 0 for an invalid request.  error: one uint64, ~0 when every crop is CLX_OK, else the failure a
 * caller checking the whole batch reports first: (kind << 62) | (crop << 32) | (uint32_t)status, kind 0 an invalid
 * request, 1 a failed frame, 2 a trailing-bytes verdict; the smallest such value, so invalid requests before failed
 * frames before trailing bytes, each in crop order. */
void* clx_batch_crop_requests(clx_batch* b);
void* clx_batch_crop_status(clx_batch* b);
void* clx_batch_crop_lengths(clx_batch* b);
void* clx_batch_crop_error(clx_batch* b);
/* The frame a crop batch decodes in its unused slots (1 channel, 16 bits, 192 samples of CONSTANT 0, valid CRC-8 and
 * CRC-16), for inspection: writes it into out if cap suffices and returns its length in bytes.  Host only. */
size_t clx_crop_filler_frame(uint8_t* out, size_t cap);
/* Packed batches: whole files or excerpts of different lengths of a corpus, one after another along the columns of one
 * [C, max_samples] output (load()'s layout), planned on the device like a crop batch.  A call: write `count` requests
 * into clx_batch_packed_requests and the count into clx_batch_packed_count (device memory), clx_batch_decode.
 *
 * Excerpt b < count is samples [offset, offset + n_b) of its file, n_b = min(length, N - offset) (N - offset for a
 * length of -1), N the file's length.  Columns: start_0 = 0, start_{b+1} = start_b + round_up_4(n_b).  A request with
 * file >= n_files, reserved != 0, offset < 0 or > N, length 0 or below -1 is invalid and takes 0 columns; an excerpt
 * with start_b + n_b > max_samples does not fit.  Both get status CLX_ERR_INVALID_ARGUMENT, length 0 and no frames
 * (starts only grow, so the excerpts that fit are a prefix of the valid ones).  Channel c of excerpt b goes to row c,
 * columns [start_b, start_b + n_b); every other element of [C, max_samples] is 0 after the call (the batch keeps the
 * previous call's end column and zeroes only what lies between the two ends, never the whole output).  Status, lengths
 * and the error word: clx_batch_crop_status / _lengths / _error, per excerpt as for crop batches (kind 0 covers invalid
 * and non-fitting excerpts).
 * Output: C rows of clx_batch_packed_stride elements, C the corpus's largest channel count; stride = round_up_4(
 * max_samples) + W, the W = round_up_4(min(max_samples, the largest block size of the corpus and the filler frame))
 * columns after round_up_4(max_samples) take the unused slots.  Memory: C * stride output elements and, per slot, a
 * planar scratch of the corpus's largest frame, slots = clx_packed_frames_bound; over a host corpus also a staging
 * buffer of clx_packed_bytes_bound bytes plus the filler frame and slack.
 * CLX_ERR_INVALID_ARGUMENT for: max_excerpts 0 or 2^30 or more, max_samples 0, slots of 2^32 or more, sizes that
 * overflow, a mode other than the two channels modes, F32 with a frame above 24 bits. */
typedef struct clx_packed_request {
    uint32_t file;     /* index of the file in the corpus */
    uint32_t reserved; /* 0 */
    int64_t offset;    /* first sample, 0 .. the file's length */
    int64_t length;    /* >= 1, or -1: to the end of the file */
} clx_packed_request;
int clx_batch_create_packed(clx_ctx* ctx, clx_corpus* corpus, size_t max_excerpts, size_t max_samples, uint32_t mode,
                            clx_batch** out);
/* The most frames the excerpts that fit can overlap together: with k = min(max_excerpts, max_samples) and m the smallest
 * block size among the frames that are not the last of their file, floor((max_samples - 2k) / m) + 2k (rounded down),
 * at most k times the frames of the largest file; k when no file has two frames.  Host only.  0 for a bad file_frames or
 * a zero argument. */
size_t clx_packed_frames_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                               size_t max_excerpts, size_t max_samples);
/* The staging bytes of a packed batch over a host corpus: clx_packed_frames_bound times the largest per-frame byte
 * advance (a frame's distance to the next frame of its file, or its byte_len when that is larger or it is the last), plus
 * 16 per excerpt for alignment.  SIZE_MAX if that overflows.  Host only.  0 for a bad file_frames or a zero argument. */
size_t clx_packed_bytes_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                              size_t max_excerpts, size_t max_samples);
/* Shared host corpora: a corpus IMAGE is one file, written once (normally on a tmpfs such as /dev/shm), that holds a
 * host corpus's frame index and bytes; every process and GPU of a machine maps it and attaches it, so the pinned bytes
 * exist once per machine instead of once per context.  All integers little-endian, at these offsets:
 *   [0, 96)                           clx_image_header
 *   [files_offset, + files_bytes)     clx_image_file (88 bytes) per file; files_offset = 128
 *   [descs_offset, + (n_frames+1)*40) clx_frame_desc: the corpus's frames, file by file in stream order, byte_offset
 *                                     relative to the bytes region and out_offset 0, then the filler frame of
 *                                     clx_crop_filler_frame (byte_offset nbytes, its exact byte_len, flags
 *                                     CLX_FRAME_CRC16_VERIFIED); descs_offset = files_offset + files_bytes rounded up
 *                                     to 64
 *   [bytes_offset, + bytes_size)      the bytes region, as a host corpus holds it: each file's bytes from its first frame
 *                                     to its end, back to back (nbytes in all), the filler frame, zeros up to
 *                                     bytes_size = round_up_64(nbytes + filler length) + 128; bytes_offset =
 *                                     descs_offset + descs_bytes rounded up to CLX_IMAGE_ALIGN
 * total_bytes = bytes_offset + bytes_size, and every gap between sections is zero.  Only the bytes region is read
 * after attaching; the header, file records and descriptors are copied (validated) once.
 *
 * clx_corpus_image_bytes: the size of the image of n_files files, file i being file_nbytes[i] bytes whose frames are
 * descs[file_frames[i] .. file_frames[i + 1]) with byte_offset into that file; 0 for a bad file_frames, a first frame
 * past its file's end, or a size that overflows.  Host only.
 * clx_corpus_image_write: writes that image into image[0, image_bytes), image_bytes being exactly that size, copying
 * file i's bytes straight from file_bytes[i] (e.g. its memory map) and infos[i] into its record.  It refuses
 * (CLX_ERR_INVALID_ARGUMENT) what clx_corpus_create_ex(..., CLX_CORPUS_HOST) refuses, each file's frames checked
 * against its own buffer, and a file_frames[0] other than 0 (frames outside every file); it computes each file's trailing-bytes verdict once, as clx_corpus_create_ex does (a file
 * whose last frame lacks CLX_FRAME_CRC16_VERIFIED has that frame decoded on the context's device).  The magic is
 * stored last, so an image whose magic reads right was written through.
 * clx_corpus_image_check: CLX_OK if image[0, image_bytes) is a well-formed image, else CLX_ERR_INVALID_ARGUMENT: the
 * magic, version, header size, counts (below 2^32 - 1), every offset and size against the layout above, image_bytes ==
 * total_bytes, the gaps and padding zero, the filler frame and its descriptor, each frame as the create calls check it
 * and inside its file's bytes, each file's frames in byte order with one channel count, starting at its byte_base, the
 * files' bytes and frame ranges back to back, flags and verdicts as the writer sets them.  Host only; no context.
 * clx_corpus_attach: checks the image, registers its bytes region with cudaHostRegister (mapped, portable), uploads the
 * frame index, and returns a host corpus over those pages: crop and packed batches, clx_corpus_device_bytes (the index
 * only) and clx_corpus_destroy work on it as on any CLX_CORPUS_HOST corpus, with the same results.  The registration is
 * counted in a process-wide registry keyed by address and length, so contexts of one process, on one device or on
 * several, can attach the same mapping; the last destroy unregisters it (destroy never frees the image, which belongs to
 * the caller and must stay mapped until then).  A refused or failed attach leaves nothing registered.  The mapping must
 * be writable (the driver pins pages writable); the library never writes to it.  If the bytes region changes after
 * attaching, the crops that read the changed bytes get wrong samples or a CRC error, never an access outside the
 * region: every span comes from the index copied at attach time. */
#define CLX_IMAGE_MAGIC 0x3150524f43584c43ull /* the bytes "CLXCORP1" */
#define CLX_IMAGE_VERSION 1u
#define CLX_IMAGE_ALIGN 4096u
#define CLX_IMAGE_END_CONFIRMED 1u /* clx_image_file.flags: the file has no frames, or its last frame's end is confirmed */
typedef struct clx_image_header {
    uint64_t magic;          /* CLX_IMAGE_MAGIC */
    uint32_t version;        /* CLX_IMAGE_VERSION */
    uint32_t header_bytes;   /* sizeof(clx_image_header) = 96 */
    uint64_t n_files, n_frames;
    uint64_t files_offset, files_bytes;  /* n_files * sizeof(clx_image_file) */
    uint64_t descs_offset, descs_bytes;  /* (n_frames + 1) * sizeof(clx_frame_desc) */
    uint64_t bytes_offset, bytes_size;
    uint64_t nbytes;         /* the files' bytes at the start of the region */
    uint64_t total_bytes;
} clx_image_header;
typedef struct clx_image_file {
    clx_streaminfo info;     /* as given to the writer */
    uint64_t byte_base;      /* where the file's bytes start in the region: the sum of the byte_counts before it */
    uint64_t byte_count;     /* its bytes from its first frame to its end; 0 for a file without frames */
    uint32_t first_frame;    /* its frames are descriptors [first_frame, first_frame + n_frames) */
    uint32_t n_frames;
    uint32_t flags;          /* CLX_IMAGE_END_CONFIRMED or 0 */
    int32_t tail;            /* trailing-bytes verdict: CLX_OK, or a frame header status 2..10 when the end is unconfirmed */
} clx_image_file;
size_t clx_corpus_image_bytes(const size_t* file_nbytes, const clx_frame_desc* descs, size_t n_frames,
                              const uint32_t* file_frames, size_t n_files);
int clx_corpus_image_write(clx_ctx* ctx, const uint8_t* const* file_bytes, const size_t* file_nbytes,
                           const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                           const clx_streaminfo* infos, void* image, size_t image_bytes);
int clx_corpus_image_check(const void* image, size_t image_bytes);
int clx_corpus_attach(clx_ctx* ctx, void* image, size_t image_bytes, clx_corpus** out);
/* Device pointers of a packed batch (NULL for other batches): max_excerpts requests (zeroed at creation); one uint32, how
 * many of them a call uses (0 at creation); max_excerpts int64 column starts, written by each call.  The row stride of
 * the output in elements (0 for other batches). */
void* clx_batch_packed_requests(clx_batch* b);
void* clx_batch_packed_count(clx_batch* b);
void* clx_batch_packed_starts(clx_batch* b);
size_t clx_batch_packed_stride(clx_batch* b);
/* Resampled crop batches: crop batches of a corpus whose files may have different sample rates, every crop at one
 * target rate R.  file_rates[i] is file i's rate r_i (its STREAMINFO sample_rate); n_files must be the corpus's.  Crop b
 * of request {file, 0, offset} is resample(x, r, R)[:, offset : offset + num_frames], x the whole file, where resample is
 * torchaudio.functional.resample with its defaults (lowpass_filter_width 6, rolloff 0.99, sinc_interp_hann): with g =
 * gcd(r, R), o = r / g, n = R / g, base = min(o, n) * 0.99 and w = ceil(6 * o / base), output j = blk * n + ph is
 * sum h[ph, k] * x[blk * o + k] over k in [-w, w + o), samples outside the file reading 0, h = sinc(t) * cos(t * pi /
 * 12)^2 * base / o with t = (k / o - ph / n) * base (taps with |t| >= 6 are skipped); N_t = ceil(N * n / o) outputs.
 * A file with r == R is copied, not filtered (N_t = N), bit for bit what clx_batch_create_crops gives.
 * The output is [n_crops * C, num_frames] float32 (CLX_OUT_CHANNELS_F32), C the corpus's largest channel count.  The
 * crop accessors serve the batch: requests (clx_crop_request, offsets at rate R), status, lengths (min(num_frames, N_t -
 * offset), 0 for an invalid request), error and clx_batch_device_out.  A request with file >= n_files, reserved != 0,
 * offset < 0 or > N_t is invalid (status CLX_ERR_INVALID_ARGUMENT, kind 0 in the error word, zero rows); a valid crop's
 * status and error word are those of a crop of its source span: the samples its outputs read, clipped to the file.
 * Columns past a crop's length and rows its file does not have read 0.
 * Each call decodes every crop's source span with the launch sequence of a packed batch, sized so that every span fits
 * (n_crops columns of round_up_4 of the largest clx_resample_source_bound over the corpus's rates), between a kernel
 * that maps the requests to source spans and the filter kernel, which writes every element of the output.
 * CLX_ERR_INVALID_ARGUMENT for: a rate or target rate of 0 or above CLX_MAX_SAMPLE_RATE, more than 2^24 filter
 * coefficients over the distinct rates (n times the taps per phase each), what clx_batch_create_packed refuses for that
 * size in CLX_OUT_CHANNELS_F32 (frames above 24 bits among them), n_crops 0 or 2^30 or more, num_frames 0, sizes that
 * overflow. */
#define CLX_MAX_SAMPLE_RATE 655350u
int clx_batch_create_resampled_crops(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                                     size_t n_crops, size_t num_frames, uint32_t target_rate, clx_batch** out);
/* The most source samples a resampled crop of num_frames outputs reads from a file of rate orig: num_frames when orig ==
 * target, else (floor((num_frames - 1) / n) + 2) * o + 2w.  SIZE_MAX if that overflows; 0 for a zero argument or a rate
 * above CLX_MAX_SAMPLE_RATE.  Host only. */
size_t clx_resample_source_bound(uint32_t orig, uint32_t target, size_t num_frames);
/* Resampled packed batches: packed batches of a corpus whose files may have different sample rates, every excerpt at one
 * target rate R, with the filter of clx_batch_create_resampled_crops.  Everything counts samples at R: offsets, lengths,
 * max_samples (T), the column starts and the returned lengths.  Excerpt b of request {file, 0, offset, length} is
 * resample(x, r, R)[:, offset : offset + n_b], x the whole file, with n_b = min(length, N_t - offset) (N_t - offset for
 * a length of -1); so the samples near an excerpt's edges are those of the resampled file.  The layout is
 * clx_batch_create_packed's: start_0 = 0 and start_{b+1} = start_b + round_up_4(n_b) over the valid requests, those
 * that do not fit included.  A request with file >= n_files, reserved != 0, offset < 0 or > N_t, or a length of 0 or
 * below -1 is invalid; an excerpt with start_b + n_b > T does not fit; both get status CLX_ERR_INVALID_ARGUMENT, length
 * 0, no columns and kind 0 in the error word.  offset == N_t is the valid empty excerpt.  A valid excerpt's status is
 * that of its source span, as for resampled crops.  A file with r == R is copied, not filtered: over a corpus whose
 * files are all at R, output, starts, lengths, status and error word are clx_batch_create_packed's (CLX_OUT_CHANNELS_F32)
 * bit for bit.
 * The output is [C, stride] float32 with stride = round_up_4(T); every element no excerpt covers reads 0 after every
 * call (alignment gaps, rows a file does not have, the columns past the last excerpt and [T, stride)).  The packed
 * accessors return the batch's own requests (clx_packed_request at rate R), count and target column starts, and the
 * stride; clx_batch_crop_status / _error return the inner packed batch's, clx_batch_crop_lengths the lengths at R.
 * Each call runs a kernel that lays the excerpts out at R and maps each one that fits to its source span, the launch
 * sequence of an inner packed batch of clx_resample_packed_source_bound columns, and the filter kernel, which writes
 * every element of the output.  CLX_ERR_INVALID_ARGUMENT for what clx_batch_create_resampled_crops refuses (its rates,
 * its coefficient limit, sizes that overflow), for what clx_batch_create_packed refuses at the inner batch's size, and
 * for max_excerpts 0 or 2^30 or more and max_samples 0. */
int clx_batch_create_resampled_packed(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                                      size_t max_excerpts, size_t max_samples, uint32_t target_rate, clx_batch** out);
/* The inner packed batch's columns of a resampled packed batch: at least sum_b round_up_4(span_b) over any excerpts
 * that fit in max_samples (T) columns at target_rate, span_b an excerpt's source span.  An excerpt of m >= 1 outputs has
 * round_up_4(span) <= (r / R) m + c_r, c_r = 2o + 2w + 3 for r != R and 3 for r == R, and at most k = min(max_excerpts,
 * T) excerpts have outputs, m's adding up to T at most: ceil(T * max r / R) + k * max c_r, rounded up to 4.  SIZE_MAX if
 * that overflows; 0 for a zero argument, a rate above CLX_MAX_SAMPLE_RATE or no file_rates for n_files > 0.  Host only. */
size_t clx_resample_packed_source_bound(const uint32_t* file_rates, size_t n_files, uint32_t target_rate,
                                        size_t max_excerpts, size_t max_samples);
/* Mel crop batches: the mel spectrogram of every row of a crop batch, torchaudio.transforms.MelSpectrogram with power
 * 2, normalized False, pad 0, onesided and pad_mode "reflect", optionally followed by a natural log.  The inner batch is
 * clx_batch_create_crops(ctx, corpus, n_crops, num_frames, CLX_OUT_CHANNELS_F32) when target_rate is 0 (file_rates may
 * then be NULL), else clx_batch_create_resampled_crops(ctx, corpus, file_rates, n_files, n_crops, num_frames,
 * target_rate); x is its [n_crops * C, L] output (L = num_frames), zero columns and rows included.  For each row: with
 * CLX_MEL_CENTER it is reflect-padded by n_fft / 2 on each side with its own samples, and F = 1 + L / hop_length; else
 * F = 1 + (L - n_fft) / hop_length.  Frame t is samples [t * hop, t * hop + n_fft) of the (padded) row times the
 * window's win_length values at offset (n_fft - win_length) / 2, zeros around them; mel[m, t] = sum_k fbank[k * n_mels
 * + m] |X_t[k]|^2 over k <= n_fft / 2, X_t the DFT of the frame (fbank: torchaudio's melscale_fbanks layout, [n_fft / 2
 * + 1][n_mels]); with CLX_MEL_LOG the output is ln(max(mel, log_floor)), ln(log_floor) taken in float64.  The output is
 * [n_crops * C, n_mels, F] float32, element (r, m, t) at (r * n_mels + m) * F + t, written whole by each call: an
 * invalid request's features are 0 (ln(log_floor) with the log), a failed crop's are unspecified.  The crop accessors
 * (requests, status, lengths in samples at the crop's rate, error) return the inner batch's buffers;
 * clx_batch_device_out, decode, sync, last_kernel_ms, read_to and clx_ctx_run_steps work on the mel batch.  Each call is
 * the inner batch's launch sequence and one more kernel, which reads the inner output once per frame overlap and keeps
 * the FFTs in shared memory: the batch holds the inner batch, the output and tables of a few times n_fft floats.  The
 * power is computed in f32 from float64 tables, each mel summing only its bins of non-zero weight.
 * CLX_ERR_INVALID_ARGUMENT for what the inner create refuses; NULL params, window or fbank; n_fft odd, below 8, above
 * 4096 or with n_fft / 2 having a prime factor above 5; win_length 0 or above n_fft; hop_length 0; n_mels 0 or above
 * 512; other flags; with CLX_MEL_LOG a log_floor that is not finite and > 0, without it one that is not 0; a window or
 * fbank value that is not finite; num_frames <= n_fft / 2 with CLX_MEL_CENTER (torch.stft refuses that reflect pad),
 * num_frames < n_fft without; sizes that overflow.
 * Normalised features: with CLX_MEL_NORM_PER_FEATURE or CLX_MEL_NORM_WHISPER (each needs CLX_MEL_LOG and
 * CLX_MEL_CENTER; not both) one more kernel, mel_norm_kernel, rewrites the log features in place after the mel kernel,
 * each reduction and map in float64 with one rounding to float32, in a fixed order without atomics.
 * CLX_MEL_NORM_PER_FEATURE: for each (crop b, row, mel), x its first v_b frames with v_b = 1 + n_b / hop_length (n_b
 * the crop's length in samples; v_b = 0 when n_b = 0), mu = mean(x), sigma = sqrt(sum (x - mu)^2 / (v_b - 1)) (0 when
 * v_b = 1) and y = (x - mu) / (sigma + 1e-5): NeMo's per_feature normalize_batch with torch.stft's frame count.  Frames
 * t >= v_b read exactly 0, so an invalid crop is all 0, and so are rows its file does not have (constant features).
 * CLX_MEL_NORM_WHISPER: the output has F' = F - 1 frames (Whisper drops the last STFT frame; the kept frames are those
 * of the unnormalised batch bit for bit) and, with l = x / ln 10 and M the largest l of the row's [n_mels, F'], y =
 * (max(l, M - 8) + 4) / 4: WhisperFeatureExtractor's log-mel of the crop as its zero-padded input.  Refused when F < 2.
 * Each call is then the inner batch's launch sequence and two kernels.  Also CLX_ERR_INVALID_ARGUMENT for a
 * normalisation flag without both CLX_MEL_LOG and CLX_MEL_CENTER, for both flags, and for CLX_MEL_NORM_PER_FEATURE with
 * n_crops * C * n_mels (max_excerpts * C * n_mels for packed batches) of 2^31 or more. */
#define CLX_MEL_CENTER 1u  /* reflect-pad n_fft / 2 samples on each side (torch.stft center=True, pad_mode "reflect") */
#define CLX_MEL_LOG 2u     /* store ln(max(mel, log_floor)) */
#define CLX_MEL_NORM_PER_FEATURE 4u  /* per-(crop or excerpt, row, mel) mean / variance over the valid frames */
#define CLX_MEL_NORM_WHISPER 8u      /* Whisper's clamp to the row's max - 8 in log10 and (l + 4) / 4; crops only */
typedef struct clx_mel_params {
    uint32_t n_fft;       /* even, 8 .. 4096, n_fft / 2 with no prime factor above 5 (400, 512, 320, 480, 1024, 2048 ...) */
    uint32_t win_length;  /* 1 .. n_fft */
    uint32_t hop_length;  /* >= 1 */
    uint32_t n_mels;      /* 1 .. 512 */
    uint32_t flags;       /* CLX_MEL_* */
    float log_floor;      /* > 0 and finite with CLX_MEL_LOG, else 0 */
} clx_mel_params;
int clx_batch_create_mel_crops(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                               size_t n_crops, size_t num_frames, uint32_t target_rate, const clx_mel_params* params,
                               const float* window /* win_length */, const float* fbank /* [n_fft / 2 + 1][n_mels] */,
                               clx_batch** out);
/* Mel packed batches: the mel spectrogram of every excerpt of a packed batch, packed along frames.  The inner batch is
 * clx_batch_create_packed(ctx, corpus, max_excerpts, max_samples, CLX_OUT_CHANNELS_F32) when target_rate is 0 (file_rates
 * may then be NULL), else clx_batch_create_resampled_packed(ctx, corpus, file_rates, n_files, max_excerpts, max_samples,
 * target_rate); x is its [C, stride] output, s_b and n_b excerpt b's sample start and length.  Excerpt b's frames are
 * clx_batch_create_mel_crops's transform of the row slices x[:, s_b : s_b + n_b], each reflect-padded with its own
 * samples at its own two edges, with the same params, window and fbank: F_b = 1 + n_b / hop_length when n_b > n_fft / 2
 * with CLX_MEL_CENTER, 1 + (n_b - n_fft) / hop_length when n_b >= n_fft without, else 0.  So an invalid, non-fitting,
 * empty or unused excerpt (n_b = 0) has no frames, and so has one too short for a frame: its status and length stay the
 * inner batch's.  Rows its file does not have are zeros in x and are transformed like the others (exactly 0, or
 * ln(log_floor) with CLX_MEL_LOG).  Layout: start_0 = 0, start_{b+1} = start_b + round_up_4(F_b); the output is [C,
 * n_mels, T_f] float32, T_f = clx_mel_packed_frames_bound(params, max_excerpts, max_samples), element (c, m, t) at (c *
 * n_mels + m) * T_f + t, and excerpt b's frames are columns [start_b, start_b + F_b).  Every other element reads 0 after
 * every call, with or without the log: alignment gaps and every column past the call's last excerpt.  T_f holds the
 * frames of any excerpts that fit the inner batch, so the fit rule is the packed batch's alone.  Each call is the inner
 * batch's launch sequence and two kernels: one CTA that counts and lays out the frames (device memory, written by each
 * call for b < count: clx_batch_mel_frames, int64 F_b; clx_batch_packed_starts, int64 start_b), and one CTA per (tile of
 * frame columns, row) that runs the windowing, FFT, power and mel sums of clx_batch_create_mel_crops once per tile,
 * whatever the excerpts it spans.  No atomics: calls are bit-identical.  Accessors: clx_batch_packed_requests and _count
 * are the inner batch's (requests at the inner batch's rate); clx_batch_crop_status, _lengths (samples) and _error are
 * the inner batch's; clx_batch_packed_stride is T_f; clx_batch_device_out the features.  Memory: the inner batch, C *
 * n_mels * T_f floats, 16 bytes per excerpt and tables of a few times n_fft floats.
 * CLX_ERR_INVALID_ARGUMENT for what the inner create refuses; every parameter clx_batch_create_mel_crops refuses (NULL
 * params, window or fbank, n_fft, win_length, hop_length, n_mels, flags, log_floor, non-finite window or fbank values);
 * max_excerpts 0 or 2^30 or more, max_samples 0; sizes that overflow; CLX_MEL_NORM_WHISPER (Whisper's input is a fixed
 * window).  No length is refused: a too short excerpt has 0 frames.
 * With CLX_MEL_NORM_PER_FEATURE, each (excerpt b, row c, mel m) of F_b > 0 frames is normalised over those F_b frames
 * as clx_batch_create_mel_crops normalises a crop's valid frames; the layout, starts and frame counts do not change and
 * every other element still reads 0.  Each call then runs a third kernel, one warp per (excerpt, row, mel). */
int clx_batch_create_mel_packed(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                                size_t max_excerpts, size_t max_samples, uint32_t target_rate,
                                const clx_mel_params* params, const float* window /* win_length */,
                                const float* fbank /* [n_fft / 2 + 1][n_mels] */, clx_batch** out);
/* The frame columns T_f of a mel packed batch: at least sum_b round_up_4(F_b) over any excerpts that fit in max_samples
 * (T) columns of max_excerpts (B), a multiple of 4.  With m the shortest length that has a frame (n_fft / 2 + 1 with
 * CLX_MEL_CENTER, n_fft without) and k = min(B, (T - m) / round_up_4(m) + 1) the most excerpts with frames that fit:
 * round_up_4(floor(T / hop_length) + 4k), and 0 when T < m.  SIZE_MAX if that overflows.  0 also for params that
 * clx_batch_create_mel_crops refuses, CLX_MEL_NORM_WHISPER, or a zero argument; CLX_MEL_NORM_PER_FEATURE does not
 * change it.  Host only; no context. */
size_t clx_mel_packed_frames_bound(const clx_mel_params* params, size_t max_excerpts, size_t max_samples);
/* Device pointer of a mel packed batch's max_excerpts int64 frame counts F_b (NULL for other batches). */
void* clx_batch_mel_frames(clx_batch* b);
int clx_batch_decode(clx_ctx* ctx, clx_batch* b, uint32_t stream_index); /* async on an internal stream */
int clx_batch_sync(clx_ctx* ctx, clx_batch* b);
/* Planar batches only (CLX_ERR_INVALID_ARGUMENT for any other mode). */
int clx_batch_read(clx_ctx* ctx, clx_batch* b, int32_t* out, size_t out_elems, clx_frame_result* results);
/* Any mode: copies min(out_elems, the batch's out_elems) samples of the batch's own element size into `out` and the
 * per-frame results (caller's frame order, CRC-16 verdicts applied) as clx_batch_read does. */
int clx_batch_read_to(clx_ctx* ctx, clx_batch* b, void* out, size_t out_elems, clx_frame_result* results);
void clx_batch_destroy(clx_ctx* ctx, clx_batch* b);
/* Steady-state throughput: decodes `steps` batches back to back (step i = batches[i % n_batches]
 * on internal stream i % n_streams, so several batches are in flight) and returns the device time
 * from first launch to last completion, measured with CUDA events. */
int clx_ctx_run_steps(clx_ctx* ctx, clx_batch** batches, size_t n_batches, uint32_t steps, uint32_t n_streams,
                      float* total_ms);
/* Raw device pointers of a batch (for zero-copy consumers, e.g. torch / NCCL); the output in the batch's mode. */
void* clx_batch_device_out(clx_batch* b);
void* clx_batch_device_bytes(clx_batch* b);
/* Events-based timing of the kernels of the last `clx_batch_decode` on this batch (ms). */
int clx_batch_last_kernel_ms(clx_ctx* ctx, clx_batch* b, float* ms);
/* Kernel launches issued by this context so far (bench.py's gpu_launches). */
uint64_t clx_ctx_launch_count(const clx_ctx* ctx);
void* clx_ctx_stream(clx_ctx* ctx, uint32_t stream_index); /* cudaStream_t */

/* Pinned (page-locked) host memory so that the copies inside clx_decode_frames are truly
 * asynchronous; optional — any host pointer works. */
void* clx_host_alloc(size_t bytes);
void clx_host_free(void* p);

/* ------------------------------------------------------------------------- */
/* claxon-shaped reader facade (FlacReader / FrameReader over the calls above) */
/* ------------------------------------------------------------------------- */
typedef struct clx_reader clx_reader;

/* FrameReader::new over an in-memory span positioned at a frame header
 * (src/frame.rs:652); `clx_reader_open_flac` is FlacReader::new + blocks(). */
int clx_reader_open_frames(clx_ctx* ctx, const uint8_t* bytes, size_t n, clx_reader** out);
int clx_reader_open_flac(clx_ctx* ctx, const uint8_t* bytes, size_t n, clx_reader** out);
int clx_reader_streaminfo(const clx_reader* r, clx_streaminfo* si);
/* read_next_or_eof: decodes ONE frame through the device path.  `buffer`/`capacity`
 * is the recycled Vec<i32>; on CLX_OK the block_size / channels / time outputs describe
 * the Block and `buffer[0 .. channels*block_size)` holds it.  If capacity is too small the
 * call returns CLX_ERR_INVALID_ARGUMENT with block_size and channels set, consuming nothing.
 * CLX_EOF == Ok(None). */
int clx_reader_next(clx_reader* r, int32_t* buffer, size_t capacity, uint32_t* block_size,
                    uint32_t* channels, uint64_t* time);
/* Batched extension, step 1 (optional): demuxes up to max_frames frames ahead of the reader's
 * position WITHOUT decoding and reports how many were found and how many output elements
 * clx_reader_next_batch(max_frames) needs for all of them (each frame aligned to 4 elements).
 * The demux is cached: the following next_batch with the same max_frames does not repeat it.
 * CLX_EOF at a clean end of stream; a header-level error if the very first frame has one. */
int clx_reader_plan_batch(clx_reader* r, size_t max_frames, size_t* n_frames, uint64_t* out_elems);
/* Batched extension: demuxes up to max_frames frames ahead and decodes them in one
 * device launch.  Frames that do not fit `capacity` are left for the next call; if not even the
 * first one fits the call returns CLX_ERR_INVALID_ARGUMENT (size the buffer with plan_batch).  Stops before the first frame that fails (that frame's status is
 * returned by the next call).  Returns the number of frames decoded in *n_decoded. */
int clx_reader_next_batch(clx_reader* r, size_t max_frames, int32_t* buffer, size_t capacity,
                          clx_frame_desc* descs, size_t* n_decoded);
uint64_t clx_reader_position(const clx_reader* r); /* byte offset of the next frame */
void clx_reader_close(clx_reader* r);

#ifdef __cplusplus
}
#endif
#endif /* CLAXON_B200_H */
