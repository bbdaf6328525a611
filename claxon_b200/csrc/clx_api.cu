// clx_api.cu — the device half of the C ABI (include/claxon_b200.h): context, device-resident
// batches, the end-to-end host-buffer decode call and the claxon-shaped reader facade.
//
// There is deliberately no CPU decode path in this library: without a usable CUDA device
// every entry point below fails with CLX_ERR_NO_DEVICE / CLX_ERR_CUDA.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_mel.h"

// A few long-lived host threads for the frame CRC-16 pass of batch creation from host bytes (precompute_crc):
// spawning std::threads per batch costs more than the checksums themselves (6 MB per C2 batch).
class HostPool {
public:
    explicit HostPool(unsigned n) {
        for (unsigned i = 0; i < n; i++) workers_.emplace_back([this, i] { loop(i); });
    }
    ~HostPool() {
        {
            std::lock_guard<std::mutex> g(m_);
            stop_ = true;
            gen_++;
        }
        cv_.notify_all();
        for (auto& t : workers_) t.join();
    }
    unsigned size() const { return (unsigned)workers_.size(); }
    // Runs fn(part, parts) for part = 0 .. parts-1: part 0 on the caller, the rest on the workers.
    void run(unsigned parts, const std::function<void(unsigned, unsigned)>& fn) {
        parts = std::max(1u, std::min(parts, size() + 1));
        if (parts > 1) {
            std::lock_guard<std::mutex> g(m_);
            fn_ = &fn;
            parts_ = parts;
            pending_ = parts - 1;
            gen_++;
        }
        if (parts > 1) cv_.notify_all();
        fn(0, parts);
        if (parts > 1) {
            std::unique_lock<std::mutex> l(m_);
            done_.wait(l, [this] { return pending_ == 0; });
            fn_ = nullptr;
        }
    }

private:
    void loop(unsigned idx) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(unsigned, unsigned)>* fn;
            unsigned parts;
            {
                std::unique_lock<std::mutex> l(m_);
                cv_.wait(l, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
                fn = fn_;
                parts = parts_;
            }
            if (fn && idx + 1 < parts) {
                (*fn)(idx + 1, parts);
                std::lock_guard<std::mutex> g(m_);
                if (--pending_ == 0) done_.notify_one();
            }
        }
    }
    std::vector<std::thread> workers_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    const std::function<void(unsigned, unsigned)>* fn_ = nullptr;
    unsigned parts_ = 0, pending_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
};

// The size of a device buffer for `nbytes` frame bytes: whole 64-byte TMA chunks + 128 bytes of look-ahead
// (clx::DecodeBuffers' contract).
size_t clx::padded_bytes(size_t nbytes) { return ((nbytes + 63) & ~(size_t)63) + 128; }

namespace {
using clx::padded_bytes;

bool is_channels(uint32_t mode) { return mode == CLX_OUT_CHANNELS_I32 || mode == CLX_OUT_CHANNELS_F32; }

// What one decode needs: `nbytes` frame bytes (before padding), `n_frames` frames, `planar` elements of planar i32
// output or scratch, and unless in CLX_OUT_PLANAR_I32, `conv` elements of output in `mode` and with `mark` a mark byte
// per frame (device-resident batches: their lane-per-frame decode writes `conv` itself).
struct DecodeNeed {
    size_t nbytes, n_frames, planar;
    uint32_t mode;
    size_t conv;
    bool mark;
    clx::Plan plan;
};

// Owns the device buffers of one decode, which clx::DecodeBuffers views, and is the only code that knows their sizes.
// A batch sizes them once, exactly; the host-buffer call keeps one set per stream and only ever grows it.  Borrowed
// frame bytes (a crop batch's over a device corpus) are neither allocated nor freed here.
struct DecodeStorage {
    uint8_t* bytes = nullptr; size_t buf_bytes = 0, bytes_cap = 0;
    bool borrowed = false;
    clx_frame_desc* descs = nullptr; size_t descs_cap = 0;
    int32_t* out = nullptr; size_t out_cap = 0;
    clx_frame_result* results = nullptr; size_t results_cap = 0;
    int* flags = nullptr;
    uint8_t* params = nullptr; size_t params_cap = 0;
    uint8_t* conv = nullptr; size_t conv_cap = 0;
    uint8_t* mark = nullptr; size_t mark_cap = 0;
    uint64_t* cols = nullptr; size_t cols_cap = 0;
    uint32_t* wins = nullptr; size_t wins_cap = 0;

    void borrow(uint8_t* p, size_t padded) { bytes = p; buf_bytes = padded; borrowed = true; }

    // Makes every buffer `n` asks for large enough.  !grow (a batch): exactly as large, zeroing the frame bytes, and in
    // a channels mode the output (elements no window covers read 0).  grow (the host-buffer call): a buffer that is too
    // small is reallocated with headroom, and nothing is zeroed.
    cudaError_t fit(const DecodeNeed& n, bool grow) {
        const bool channels = is_channels(n.mode);
        const size_t frames = std::max<size_t>(1, n.n_frames);
        const size_t conv_bytes = (n.conv + 8) * clx::output_elem_size(n.mode);
        cudaError_t e = cudaSuccess;
        if (!borrowed) {
            buf_bytes = padded_bytes(n.nbytes);
            e = fit_one(bytes, bytes_cap, buf_bytes, 4096, grow);
            if (e == cudaSuccess && !grow) e = cudaMemset(bytes, 0, buf_bytes);
        }
        if (e == cudaSuccess) e = fit_one(descs, descs_cap, frames, 64, grow);
        if (e == cudaSuccess) e = fit_one(out, out_cap, n.planar + 4, 4096, grow);
        if (e == cudaSuccess) e = fit_one(results, results_cap, frames, 64, grow);
        if (e == cudaSuccess && !flags) e = cudaMalloc((void**)&flags, 4 * sizeof(int));
        if (e == cudaSuccess) e = fit_one(params, params_cap, clx::coop_params_bytes(n.plan, (uint32_t)n.n_frames) + 16, 4096, grow);
        if (e == cudaSuccess && n.mode != CLX_OUT_PLANAR_I32) e = fit_one(conv, conv_cap, conv_bytes, 4096, grow);
        if (e == cudaSuccess && channels && !grow) e = cudaMemset(conv, 0, conv_bytes);
        if (e == cudaSuccess && n.mark && n.mode != CLX_OUT_PLANAR_I32) e = fit_one(mark, mark_cap, frames, 0, grow);
        if (e == cudaSuccess && channels) e = fit_one(cols, cols_cap, frames, 0, grow);
        if (e == cudaSuccess && channels) e = fit_one(wins, wins_cap, frames, 0, grow);
        return e;
    }

    clx::DecodeBuffers view(uint32_t n_frames, uint32_t mode, uint64_t stride) const {
        return clx::DecodeBuffers{bytes, buf_bytes, descs, n_frames, out, results, flags, params, mode, conv, mark, cols,
                                  stride, wins};
    }

    void release() {
        if (!borrowed) cudaFree(bytes);
        cudaFree(descs); cudaFree(out); cudaFree(results); cudaFree(flags); cudaFree(params);
        cudaFree(conv); cudaFree(mark); cudaFree(cols); cudaFree(wins);
    }

private:
    // `p` holds at least `need` elements afterwards: when it had to be reallocated, exactly that many, or with `grow`
    // a quarter more plus `slack`.
    template <typename T>
    static cudaError_t fit_one(T*& p, size_t& cap, size_t need, size_t slack, bool grow) {
        if (p && need <= cap) return cudaSuccess;
        cudaError_t e = cudaFree(p);
        p = nullptr; cap = 0;
        const size_t want = grow ? need + need / 4 + slack : need;
        if (e == cudaSuccess) e = cudaMalloc((void**)&p, want * sizeof(T));
        if (e == cudaSuccess) cap = want;
        return e;
    }
};
}  // namespace

struct clx_ctx {
    int device = 0;
    uint32_t flags = 0;
    std::vector<cudaStream_t> streams;
    std::string last_error;
    uint64_t launches = 0;
    std::vector<DecodeStorage> scratch;  // clx_decode_frames: one grow-only set per stream (chunk pipelining)
    // pinned staging for the small per-frame tables: pageable memory would make the "async" copies
    // synchronous and serialise the chunk pipeline
    clx_frame_desc* h_descs = nullptr; size_t h_descs_cap = 0;   // rebased descriptors (H2D)
    clx_frame_result* h_results = nullptr; size_t h_results_cap = 0;  // results (D2H)
    unsigned host_threads = 1;
    HostPool* pool = nullptr;   // created on first use
};

struct clx_batch {
    // What the batch decodes: frames it was given, or one of the corpus kinds (clx_batch_create_crops ... _mel_packed).
    enum class Kind { Frames, Crops, Packed, ResampledCrops, ResampledPacked, MelCrops, MelPacked };
    Kind kind = Kind::Frames;
    DecodeStorage buf;
    size_t out_elems = 0;
    uint32_t n_frames = 0;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    cudaStream_t last_stream = nullptr;
    clx::Plan plan;
    // The batch's launch sequence (flag reset + kernels) captured once as a CUDA graph: a decode is then
    // one graph launch instead of five stream operations, which matters when a step is ~25 us.
    cudaGraphExec_t graph = nullptr;
    uint64_t graph_launches = 0;   // kernel launches inside the graph
    cudaEvent_t ev_idle = nullptr; // without a graph: the previous decode of this batch has finished
    // Frame CRC-16 (src/frame.rs:752-763): the batch's bytes never change, so the checksum of every claimed
    // span is taken once, on the host, when the batch is created; clx_batch_read applies it.
    std::vector<uint8_t> crc_ok;
    std::vector<uint64_t> h_offset;
    std::vector<uint32_t> h_len;
    std::vector<uint32_t> order;   // device position -> caller's frame index (empty: identity), see shape_order()
    bool device_crc = false;       // bytes came from device memory: the CRC-16 check runs on the device, inside the graph
    // Output mode (CLX_OUT_*).  Interleaved batches hand out buf.conv; buf.out stays their planar scratch.  The
    // lane-per-frame path writes I32 / I16 into buf.conv itself (buf.mark: the frames the generic kernel took over); every
    // other path, and I24, decodes to buf.out and converts all frames inside the graph (see clx::launch_decode).
    // Channels modes: buf.conv holds out_elems = rows * stride elements, and the device descriptors' out_offset is the
    // frame's place in the planar scratch buf.out (frames packed back to back, 4-element aligned); buf.cols holds each
    // frame's window start on row 0 (row base * stride + column), and buf.wins its window (first | count << 16; full
    // windows for clx_batch_create_channels), both in the device order.
    uint32_t mode = CLX_OUT_PLANAR_I32;
    uint64_t stride = 0;
    // Corpus batches.  Crops and Packed decode frames of `corpus`: buf.bytes is the corpus's, or over a host corpus the
    // batch's own staging buffer of `staging` bytes, the filler frame after it; the planner writes buf.descs, buf.cols
    // and buf.wins in every decode (clx_crops.cu).  The other kinds wrap `inner`, whose launch sequence runs inside
    // theirs, and write their output to buf.conv.  The buffers below are the kinds' device state; a wrapper's may point
    // into its inner batch's.  `owned` lists every device allocation of the batch outside `buf`, which is all
    // clx_batch_destroy frees besides `buf` and `inner`.
    clx_corpus* corpus = nullptr;
    std::vector<void*> owned;
    clx::ExcerptBuffers ex{};
    uint64_t staging = 0;
    clx_batch* inner = nullptr;
    clx::ResampleBuffers rs{};
    clx::MelBuffers mel{};
    size_t mel_smem = 0;
    clx::MelPacked mel_packed{};
    clx::MelNorm mel_norm{};  // flags 0 without a CLX_MEL_NORM_* flag
};

struct clx_corpus {
    uint8_t* d_bytes = nullptr; size_t nbytes = 0, buf_bytes = 0;
    uint8_t* h_bytes = nullptr;        // CLX_CORPUS_HOST: the bytes in mapped pinned memory (then d_bytes is null)
    const uint8_t* d_host = nullptr;   // ... and their device address
    bool attached = false;             // clx_corpus_attach: h_bytes is an image's registered bytes region, buf_bytes long
    size_t device_bytes = 0;           // every device allocation of the corpus
    clx_frame_desc* d_descs = nullptr;  // n_frames + 1: the filler frame last
    int64_t* d_starts = nullptr;
    uint32_t* d_file_frames = nullptr;
    int64_t* d_file_len = nullptr;
    uint32_t* d_file_ch = nullptr;
    int32_t* d_file_tail = nullptr;
    uint32_t n_frames = 0, n_files = 0;
    std::vector<clx_frame_desc> descs;  // host copy, the filler frame last
    std::vector<uint32_t> file_frames;
    uint32_t channels = 1, max_bps = 0;
    int live = 0;  // crop and packed batches of this corpus
    clx::CropCorpus view(uint64_t staging) const {
        return {d_descs, d_starts, d_file_frames, d_file_len, d_file_ch, d_file_tail, n_files, n_frames, d_host,
                d_host ? staging : 0};
    }
};

namespace {

int cuda_fail(clx_ctx* ctx, cudaError_t e, const char* what) {
    if (ctx) ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
    return CLX_ERR_CUDA;
}
#define CU(ctx, call)                                              \
    do {                                                           \
        cudaError_t e_ = (call);                                   \
        if (e_ != cudaSuccess) return cuda_fail(ctx, e_, #call);   \
    } while (0)

// Host-side frame CRC-16 (src/frame.rs:752-763) for device-resident batches: their bytes never change, so the
// checksum of every claimed span is taken once, when the batch is created (the host-buffer call checks on the
// device instead, clx_crc.cu).  It takes effect only when the subframes decoded, so subframe errors keep their
// precedence over "frame CRC mismatch"; a frame that ended somewhere else than claimed gets a second look.
void precompute_crc_range(const uint8_t* bytes, const clx_frame_desc* descs, uint8_t* verdict, size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; i++) {
        const clx_frame_desc& d = descs[i];
        if (d.flags & CLX_FRAME_CRC16_VERIFIED) { verdict[i] = 1; continue; }  // demuxer already matched it
        if (d.byte_len < 2) { verdict[i] = 0; continue; }
        const uint8_t* f = bytes + d.byte_offset;
        const uint16_t stored = (uint16_t)(((uint32_t)f[d.byte_len - 2] << 8) | f[d.byte_len - 1]);
        verdict[i] = clx_crc16(f, d.byte_len - 2) == stored ? 1 : 0;
    }
}

void precompute_crc(clx_ctx* ctx, const uint8_t* bytes, const clx_frame_desc* descs, size_t n, std::vector<uint8_t>& out) {
    out.assign(n, 0);
    uint8_t* verdict = out.data();
    unsigned nt = std::min<unsigned>(ctx->host_threads, (unsigned)std::max<size_t>(1, n / 32));
    if (nt <= 1) return precompute_crc_range(bytes, descs, verdict, 0, n);
    if (!ctx->pool) ctx->pool = new HostPool(ctx->host_threads - 1);
    ctx->pool->run(nt, [&](unsigned part, unsigned parts) {
        precompute_crc_range(bytes, descs, verdict, n * part / parts, n * (part + 1) / parts);
    });
}

int finish(clx_ctx* ctx, clx_batch* b, cudaError_t e, const char* what, clx_batch** out);

// Where a create or decode call writes its `out_elems` samples.  Planar and interleaved modes: each frame from its
// out_offset on.  Channels modes: `n_rows` rows of `stride` elements; frame i stores its window windows[i] (null: every
// frame its full window at row 0) from column out_offset on.
struct Output {
    uint32_t mode;
    size_t out_elems;
    uint32_t n_rows;
    size_t stride;
    const clx_frame_window* windows;
};

// Everything the kernels assume about a call's frames (the C ABI trusts none of it): the bytes and descriptors are
// given, and each frame lies in the bytes and has a shape the kernels decode.  With `o`, each frame also fits the
// output: the mode's sample width (interleaved I16: 16 bits, I24 and channels F32: 24), and its range of out_elems, or
// in a channels mode its window, rows and columns.  Without (a corpus), the bytes alone.
bool valid_frames(const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames, const Output* o) {
    if ((!bytes && nbytes) || (!descs && n_frames)) return false;
    const bool channels = o && is_channels(o->mode);
    if (channels && (o->n_rows == 0 || o->stride == 0 || o->stride > SIZE_MAX / 4 / o->n_rows)) return false;
    const uint32_t max_bps = !o ? 32u : o->mode == CLX_OUT_INTERLEAVED_I16 ? 16u :
                             o->mode == CLX_OUT_INTERLEAVED_I24 || o->mode == CLX_OUT_CHANNELS_F32 ? 24u : 32u;
    for (size_t i = 0; i < n_frames; i++) {
        const clx_frame_desc& d = descs[i];
        const uint32_t bps = d.bits_per_sample;
        if (!(d.byte_offset <= nbytes && d.byte_len <= nbytes - d.byte_offset && d.header_len <= d.byte_len &&
              d.n_channels >= 1 && d.n_channels <= 8 && d.block_size != 0 && d.byte_len <= (1u << 28) &&
              !(d.channel_assignment >= 8 && d.n_channels != 2) && d.channel_assignment <= 10 &&
              (bps == 0 || (bps >= 4 && bps <= max_bps))))  // 0: "not in the header" -> Unsupported, as the reference
            return false;
        if (!o) continue;
        const uint64_t elems = (uint64_t)d.n_channels * d.block_size;
        if (!channels) {
            if (d.out_offset > o->out_elems || elems > o->out_elems - d.out_offset) return false;
            continue;
        }
        const clx_frame_window w = o->windows ? o->windows[i] : clx_frame_window{0, 0, d.block_size, 0};
        if (!(w.reserved == 0 && w.row <= o->n_rows && d.n_channels <= o->n_rows - w.row && w.first < d.block_size &&
              w.count != 0 && w.count <= (uint32_t)d.block_size - w.first && d.out_offset <= o->stride &&
              w.count <= o->stride - d.out_offset))
            return false;
    }
    return true;
}
}  // namespace

bool clx::corpus_frames_ok(const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames) {
    return valid_frames(bytes, nbytes, descs, n_frames, nullptr);
}

namespace {
// Copies per-frame results from the device order to the caller's frame indices: position p holds frame order[p] (an
// empty order: the same order).
void unpermute(const clx_frame_result* dev, const std::vector<uint32_t>& order, size_t n, clx_frame_result* results) {
    if (order.empty()) memcpy(results, dev, n * sizeof(clx_frame_result));
    else
        for (size_t p = 0; p < n; p++) results[order[p]] = dev[p];
}

int create_batch(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                 uint32_t batch_flags, const Output& o, clx_batch** out);

// The kernels map consecutive descriptors onto the lanes of a warp, and a warp advances at the pace of its longest
// block: frames of one shape belong next to each other.  Fills `order` (position -> frame index) with the frames
// [lo, hi) grouped by (channels, block size), stream order kept inside a group; returns false (order untouched) if
// they are all of one shape already — the usual case: a file's frames differ only in its last block.
bool shape_order(const clx_frame_desc* descs, size_t lo, size_t hi, std::vector<uint32_t>& order) {
    bool mixed = false;
    for (size_t i = lo + 1; i < hi && !mixed; i++)
        mixed = descs[i].block_size != descs[lo].block_size || descs[i].n_channels != descs[lo].n_channels;
    if (!mixed) return false;
    order.resize(hi - lo);
    for (size_t i = lo; i < hi; i++) order[i - lo] = (uint32_t)i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        const uint32_t ka = ((uint32_t)descs[a].n_channels << 16) | descs[a].block_size;
        const uint32_t kb = ((uint32_t)descs[b].n_channels << 16) | descs[b].block_size;
        return ka > kb;
    });
    return true;
}

// Chooses the decode path of a set of frames.  Two fast paths, two regimes.  The lane-per-frame path (clx_fused.cu)
// has the fewest instructions per sample and is what a stream of batches should use; but a lane walks its whole frame
// alone, so one call takes ~0.4 ms of device time however few frames it holds.  A synchronous host-buffer call with a
// few thousand frames and nothing else in flight is latency-bound: there the warp-per-frame path (clx_coop.cu: 32 lanes
// share a frame, ~0.25 ms per 1024 frames) finishes sooner and lets the PCM copy-out start earlier.  `latency_call` =
// the plan is for such a call.
// (Frames with many channels and long blocks — BASELINE.json's stress shape, 8 x 16384 — are latency-bound on either
// fast path: the index lane walks (channels - 1) * block_size Rice codes alone.  No special case.)
constexpr size_t kLatencyRegimeFrames = 4096;
clx::Plan make_plan(const clx_ctx* ctx, const clx_frame_desc* descs, size_t n, bool latency_call = false) {
    clx::Plan plan;
    plan.no_generic = (ctx->flags & CLX_OPT_NO_GENERIC) != 0;
    plan.no_wide = (ctx->flags & CLX_OPT_NO_WIDE) != 0;
    uint32_t max_ch = 0;
    for (size_t i = 0; i < n; i++) {
        plan.max_frame_elems = std::max<uint32_t>(plan.max_frame_elems, (uint32_t)descs[i].n_channels * descs[i].block_size);
        max_ch = std::max<uint32_t>(max_ch, descs[i].n_channels);
    }
    if ((ctx->flags & CLX_OPT_GENERIC_KERNEL_ONLY) || n == 0 || max_ch > 8) return plan;
    plan.channels = 1;
    while (plan.channels < max_ch) plan.channels <<= 1;  // a power of two, so that a warp holds whole frames
    if ((ctx->flags & CLX_OPT_WARP_PER_FRAME) || (latency_call && !(ctx->flags & CLX_OPT_LANE_PER_FRAME)))
        plan.path = clx::Path::WarpPerFrame;
    else
        plan.path = clx::Path::LanePerFrame;
    return plan;
}

}  // namespace

extern "C" {

int clx_ctx_create(const clx_options* opts, clx_ctx** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return CLX_ERR_NO_DEVICE;
    clx_ctx* ctx = new clx_ctx();
    ctx->device = opts ? opts->device : 0;
    ctx->flags = opts ? opts->flags : 0;
    if (ctx->device < 0 || ctx->device >= count) { delete ctx; return CLX_ERR_NO_DEVICE; }
    if (cudaSetDevice(ctx->device) != cudaSuccess) { delete ctx; return CLX_ERR_NO_DEVICE; }
    if (clx::crc16_init() != cudaSuccess) { delete ctx; return CLX_ERR_CUDA; }
    uint32_t ns = opts && opts->n_streams ? opts->n_streams : 2;
    ns = std::min<uint32_t>(ns, 128);
    ctx->streams.resize(ns);
    for (uint32_t i = 0; i < ns; i++)
        if (cudaStreamCreateWithFlags(&ctx->streams[i], cudaStreamNonBlocking) != cudaSuccess) {
            delete ctx;
            return CLX_ERR_CUDA;
        }
    ctx->scratch.resize(ns);
    ctx->host_threads = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
    if (opts && opts->host_threads) ctx->host_threads = std::max(1u, std::min(64u, opts->host_threads));
    *out = ctx;
    return CLX_OK;
}

void clx_ctx_destroy(clx_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (auto& s : ctx->scratch) s.release();
    for (auto s : ctx->streams) cudaStreamDestroy(s);
    if (ctx->h_descs) cudaFreeHost(ctx->h_descs);
    if (ctx->h_results) cudaFreeHost(ctx->h_results);
    delete ctx->pool;
    delete ctx;
}

const char* clx_ctx_last_error(const clx_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }
uint64_t clx_ctx_launch_count(const clx_ctx* ctx) { return ctx ? ctx->launches : 0; }
void* clx_ctx_stream(clx_ctx* ctx, uint32_t i) { return ctx ? (void*)ctx->streams[i % ctx->streams.size()] : nullptr; }

// ---------------------------------------------------------------------------------
// end-to-end decode with host buffers
// ---------------------------------------------------------------------------------
int clx_decode_frames(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                      size_t n_frames, int32_t* out, size_t out_elems, clx_frame_result* results) {
    return clx_decode_frames_to(ctx, bytes, nbytes, descs, n_frames, out, out_elems, results, CLX_OUT_PLANAR_I32);
}

int clx_decode_frames_to(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                         size_t n_frames, void* out_v, size_t out_elems, clx_frame_result* results, uint32_t mode) {
    const Output o{mode, out_elems, 0, 0, nullptr};
    if (!ctx || (!results && n_frames) || mode > CLX_OUT_INTERLEAVED_I24 || !valid_frames(bytes, nbytes, descs, n_frames, &o))
        return CLX_ERR_INVALID_ARGUMENT;
    if (n_frames == 0) return CLX_OK;
    uint8_t* const out = static_cast<uint8_t*>(out_v);
    const size_t esize = clx::output_elem_size(mode);
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    CU(ctx, cudaSetDevice(ctx->device));
    const double t0 = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    // Chunks of frames are pipelined over the context's streams: H2D of chunk i+1 and D2H of
    // chunk i-1 overlap the kernels of chunk i.  A chunk covers a contiguous byte range and a
    // contiguous output range (descriptors in stream order, as the demuxer emits them).
    const size_t ns = ctx->streams.size();
    size_t n_chunks = std::min<size_t>(ns, std::max<size_t>(1, n_frames / 128));
    for (size_t i = 1; i < n_frames && n_chunks > 1; i++)  // chunking needs stream order on both sides
        if (descs[i].byte_offset < descs[i - 1].byte_offset || descs[i].out_offset < descs[i - 1].out_offset)
            n_chunks = 1;
    if (ctx->h_descs_cap < n_frames) {
        if (ctx->h_descs) cudaFreeHost(ctx->h_descs);
        if (ctx->h_results) cudaFreeHost(ctx->h_results);
        ctx->h_descs = nullptr; ctx->h_results = nullptr; ctx->h_descs_cap = ctx->h_results_cap = 0;
        const size_t cap = n_frames + n_frames / 2 + 1024;
        CU(ctx, cudaHostAlloc((void**)&ctx->h_descs, cap * sizeof(clx_frame_desc), cudaHostAllocDefault));
        CU(ctx, cudaHostAlloc((void**)&ctx->h_results, cap * sizeof(clx_frame_result), cudaHostAllocDefault));
        ctx->h_descs_cap = ctx->h_results_cap = cap;
    }
    memcpy(ctx->h_descs, descs, n_frames * sizeof(clx_frame_desc));
    struct Span { size_t f0, f1; uint64_t b0, b1, o0, o1; };
    std::vector<Span> spans;
    std::vector<uint32_t> device_order;  // empty: the device sees the frames in the caller's order
    for (size_t c = 0; c < n_chunks; c++) {
        Span s{n_frames * c / n_chunks, n_frames * (c + 1) / n_chunks, ~0ull, 0, ~0ull, 0};
        for (size_t i = s.f0; i < s.f1; i++) {
            const clx_frame_desc& d = descs[i];
            s.b0 = std::min<uint64_t>(s.b0, d.byte_offset & ~15ull);
            s.b1 = std::max<uint64_t>(s.b1, d.byte_offset + d.byte_len);
            s.o0 = std::min<uint64_t>(s.o0, d.out_offset);
            s.o1 = std::max<uint64_t>(s.o1, d.out_offset + (uint64_t)d.n_channels * d.block_size);
        }
        // The device copy of the chunk's output keeps the host layout's alignment (offset mod 4 elements, so
        // 16-byte stores stay possible) but the copy back covers exactly [o0, o1): it never touches an element
        // before the chunk's first frame, so neighbouring chunks cannot overlap on the host side.
        // device order of the chunk's frames: grouped by shape (position p of the chunk holds frame order[p])
        std::vector<uint32_t> order;
        if (shape_order(descs, s.f0, s.f1, order)) {
            if (device_order.empty()) {
                device_order.resize(n_frames);
                for (size_t i = 0; i < n_frames; i++) device_order[i] = (uint32_t)i;
            }
            for (size_t p = 0; p < order.size(); p++) {
                device_order[s.f0 + p] = order[p];
                ctx->h_descs[s.f0 + p] = descs[order[p]];
            }
        }
        for (size_t i = s.f0; i < s.f1; i++) {
            ctx->h_descs[i].byte_offset -= s.b0;
            ctx->h_descs[i].out_offset -= s.o0 & ~3ull;
        }
        spans.push_back(s);
    }
    size_t enqueued = 0;  // chunks with work in flight
    // On any failure after the first enqueue: nothing may still be writing into the caller's buffers on return.
    auto drain = [&](int rc) {
        for (size_t c = 0; c < enqueued && c < n_chunks; c++) cudaStreamSynchronize(ctx->streams[c]);
        return rc;
    };
#define CUD(call)                                                         \
    do {                                                                  \
        cudaError_t e_ = (call);                                          \
        if (e_ != cudaSuccess) return drain(cuda_fail(ctx, e_, #call));   \
    } while (0)
    for (size_t c = 0; c < n_chunks; c++) {
        const Span& s = spans[c];
        DecodeStorage& sc = ctx->scratch[c];
        cudaStream_t st = ctx->streams[c];
        const size_t nb = (size_t)(s.b1 - s.b0), nf = s.f1 - s.f0, lead = (size_t)(s.o0 & 3), no = (size_t)(s.o1 - s.o0);
        const clx::Plan plan = make_plan(ctx, descs + s.f0, nf, n_frames <= kLatencyRegimeFrames);
        // (never fused: no mark; the frame CRC-16 on the device, src/frame.rs:752-763)
        CUD(sc.fit({nb, nf, lead + no, mode, lead + no, false, plan}, true));
        enqueued = c + 1;
        CUD(cudaMemcpyAsync(sc.bytes, bytes + s.b0, nb, cudaMemcpyHostToDevice, st));
        CUD(cudaMemcpyAsync(sc.descs, ctx->h_descs + s.f0, nf * sizeof(clx_frame_desc), cudaMemcpyHostToDevice, st));
        CUD(clx::launch_decode(sc.view((uint32_t)nf, mode, 0), plan, !(ctx->flags & CLX_OPT_NO_VERIFY_CRC), st, &ctx->launches));
        if (mode == CLX_OUT_PLANAR_I32)
            CUD(cudaMemcpyAsync(out + s.o0 * esize, sc.out + lead, no * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        else
            CUD(cudaMemcpyAsync(out + s.o0 * esize, sc.conv + lead * esize, no * esize, cudaMemcpyDeviceToHost, st));
        CUD(cudaMemcpyAsync(ctx->h_results + s.f0, sc.results, nf * sizeof(clx_frame_result), cudaMemcpyDeviceToHost, st));
    }
#ifdef CLX_EXPERIMENT
    static const bool trace = getenv("CLX_TRACE") != nullptr;
#else
    constexpr bool trace = false;
#endif
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t1 = trace ? now() : 0;
    for (size_t c = 0; c < n_chunks; c++) CUD(cudaStreamSynchronize(ctx->streams[c]));
#undef CUD
    const double t2 = trace ? now() : 0;
    unpermute(ctx->h_results, device_order, n_frames, results);
    if (trace)
        fprintf(stderr, "[clx] frames=%zu chunks=%zu submit=%.3f ms wait=%.3f ms results=%.3f ms\n", n_frames, n_chunks, t1 - t0,
                t2 - t1, now() - t2);
    return CLX_OK;
}

// ---------------------------------------------------------------------------------
// device-resident batches
// ---------------------------------------------------------------------------------
int clx_batch_create(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                     size_t out_elems, clx_batch** out) {
    return clx_batch_create_ex(ctx, bytes, nbytes, descs, n_frames, out_elems, 0, out);
}

int clx_batch_create_ex(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                        size_t out_elems, uint32_t batch_flags, clx_batch** out) {
    return clx_batch_create_to(ctx, bytes, nbytes, descs, n_frames, out_elems, batch_flags, CLX_OUT_PLANAR_I32, out);
}

int clx_batch_create_to(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                        size_t out_elems, uint32_t batch_flags, uint32_t mode, clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    const Output o{mode, out_elems, 0, 0, nullptr};
    if (!ctx || mode > CLX_OUT_INTERLEAVED_I24 || !valid_frames(bytes, nbytes, descs, n_frames, &o))
        return CLX_ERR_INVALID_ARGUMENT;
    return create_batch(ctx, bytes, nbytes, descs, n_frames, batch_flags, o, out);
}

int clx_batch_create_channels(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                              size_t n_frames, uint32_t n_channels, size_t channel_stride, uint32_t batch_flags,
                              uint32_t mode, clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    const Output o{mode, (size_t)n_channels * channel_stride, n_channels, channel_stride, nullptr};
    if (!ctx || n_channels > 8 || !is_channels(mode) || !valid_frames(bytes, nbytes, descs, n_frames, &o))
        return CLX_ERR_INVALID_ARGUMENT;
    return create_batch(ctx, bytes, nbytes, descs, n_frames, batch_flags, o, out);
}

int clx_batch_create_windows(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs,
                             const clx_frame_window* windows, size_t n_frames, uint32_t n_rows, size_t row_stride,
                             uint32_t batch_flags, uint32_t mode, clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    const Output o{mode, (size_t)n_rows * row_stride, n_rows, row_stride, windows};
    if (!ctx || (!windows && n_frames) || !is_channels(mode) || !valid_frames(bytes, nbytes, descs, n_frames, &o))
        return CLX_ERR_INVALID_ARGUMENT;
    return create_batch(ctx, bytes, nbytes, descs, n_frames, batch_flags, o, out);
}

}  // extern "C"

namespace {
// The part of batch creation every mode shares, for arguments valid_frames accepted.
int create_batch(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                 uint32_t batch_flags, const Output& o, clx_batch** out) {
    CU(ctx, cudaSetDevice(ctx->device));
    const size_t stride = o.stride;
    const bool on_device = (batch_flags & CLX_BATCH_BYTES_ON_DEVICE) != 0;
    clx_batch* b = new clx_batch();
    b->out_elems = o.out_elems;
    b->n_frames = (uint32_t)n_frames;
    b->plan = make_plan(ctx, descs, n_frames);
    b->mode = o.mode;
    b->stride = stride;
    // Device descriptors in the device order (shape_order); in a channels mode each frame's window start moves to
    // `cols` (row base * stride + column) and its window to `wins`, and out_offset becomes its place in the planar
    // scratch, packed back to back, so that every planar kernel runs as is.
    const bool reordered = shape_order(descs, 0, n_frames, b->order);
    std::vector<clx_frame_desc> dev;
    std::vector<uint64_t> cols;
    std::vector<uint32_t> wins;
    size_t planar_elems = o.out_elems;
    if (reordered || stride) {
        dev.resize(n_frames);
        for (size_t p = 0; p < n_frames; p++) dev[p] = descs[reordered ? b->order[p] : p];
    }
    if (stride) {
        cols.resize(n_frames);
        wins.resize(n_frames);
        planar_elems = 0;
        for (size_t p = 0; p < n_frames; p++) {
            const size_t i = reordered ? b->order[p] : p;
            const clx_frame_window w = o.windows ? o.windows[i] : clx_frame_window{0, 0, dev[p].block_size, 0};
            cols[p] = (uint64_t)w.row * stride + dev[p].out_offset;
            wins[p] = w.first | (w.count << 16);
            dev[p].out_offset = planar_elems;
            planar_elems += ((size_t)dev[p].n_channels * dev[p].block_size + 3) & ~(size_t)3;
        }
    }
    cudaError_t e = b->buf.fit({nbytes, n_frames, planar_elems, o.mode, o.out_elems, true, b->plan}, false);
    if (e == cudaSuccess && stride) e = cudaMemcpy(b->buf.cols, cols.data(), n_frames * sizeof(uint64_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && stride) e = cudaMemcpy(b->buf.wins, wins.data(), n_frames * sizeof(uint32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(b->buf.bytes, bytes, nbytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
        e = cudaMemcpy(b->buf.descs, dev.empty() ? descs : dev.data(), n_frames * sizeof(clx_frame_desc), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && !(ctx->flags & CLX_OPT_NO_VERIFY_CRC)) {
        if (on_device) b->device_crc = true;  // no host copy to checksum: clx_crc.cu, as part of every decode
        else precompute_crc(ctx, bytes, descs, n_frames, b->crc_ok);
    }
    b->h_offset.resize(n_frames);
    b->h_len.resize(n_frames);
    for (size_t i = 0; i < n_frames; i++) { b->h_offset[i] = descs[i].byte_offset; b->h_len[i] = descs[i].byte_len; }
    return finish(ctx, b, e, "clx_batch_create", out);
}

cudaError_t launch_batch(clx_batch* b, cudaStream_t st, uint64_t* launches) {
    using Kind = clx_batch::Kind;
    const clx::DecodeBuffers db = b->buf.view(b->n_frames, b->mode, b->stride);
    cudaError_t e = cudaSuccess;
    switch (b->kind) {
    case Kind::Frames:
        return clx::launch_decode(db, b->plan, b->device_crc, st, launches);
    case Kind::Crops:
        return clx::launch_excerpts<clx::CropLayout>(b->corpus->view(b->staging), b->ex, db, b->plan, b->device_crc, st,
                                                     launches);
    case Kind::Packed:
        return clx::launch_excerpts<clx::PackedLayout>(b->corpus->view(b->staging), b->ex, db, b->plan, b->device_crc,
                                                       st, launches);
    case Kind::ResampledCrops:
        e = clx::launch_resample_map<clx::CropLayout>(b->corpus->view(0), b->rs, b->ex, st, launches);
        if (e == cudaSuccess) e = launch_batch(b->inner, st, launches);
        return e == cudaSuccess ? clx::launch_resample(b->rs, st, launches) : e;
    case Kind::ResampledPacked:
        e = clx::launch_resample_map<clx::PackedLayout>(b->corpus->view(0), b->rs, b->ex, st, launches);
        if (e == cudaSuccess) e = launch_batch(b->inner, st, launches);
        return e == cudaSuccess ? clx::launch_resample_packed(b->rs, b->ex, st, launches) : e;
    case Kind::MelCrops:
        e = launch_batch(b->inner, st, launches);
        return e == cudaSuccess ? clx::launch_mel(b->mel, b->mel_norm, b->mel_smem, st, launches) : e;
    case Kind::MelPacked:
        e = launch_batch(b->inner, st, launches);
        return e == cudaSuccess ? clx::launch_mel_packed(b->mel, b->mel_packed, b->mel_norm, b->mel_smem, st, launches)
                                : e;
    }
    return cudaErrorInvalidValue;
}

// Captures the batch's launch sequence once; called from clx_batch_create so that no decode ever pays for
// (or is timed with) a graph instantiation.
void build_graph(clx_ctx* ctx, clx_batch* b) {
#ifdef CLX_EXPERIMENT
    if (getenv("CLX_NO_GRAPH")) return;
#endif
    if (b->n_frames == 0 && !b->inner) return;
    cudaStream_t st = ctx->streams[0];
    cudaGraph_t g = nullptr;
    uint64_t n = 0;
    cudaError_t e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
    if (e == cudaSuccess) {
        cudaError_t e1 = launch_batch(b, st, &n);
        e = cudaStreamEndCapture(st, &g);
        if (e1 != cudaSuccess) e = e1;
    }
    if (e == cudaSuccess && g) e = cudaGraphInstantiate(&b->graph, g, 0);
    if (g) cudaGraphDestroy(g);
    if (e != cudaSuccess || !b->graph) {
        b->graph = nullptr;
        cudaGetLastError();
    } else b->graph_launches = n;
}

// The end of every public create, after the batch's buffers were made with the first CUDA error `e`: its timing events
// and its graph, or on an error none of it (the batch is destroyed).  An inner batch is never finished: the graph of
// the batch around it launches its kernels.
int finish(clx_ctx* ctx, clx_batch* b, cudaError_t e, const char* what, clx_batch** out) {
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev_start);
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev_stop);
    if (e != cudaSuccess) {
        clx_batch_destroy(ctx, b);
        return cuda_fail(ctx, e, what);
    }
    build_graph(ctx, b);
    *out = b;
    return CLX_OK;
}

// Enqueues one decode of a device-resident batch on `st`, through the batch's graph when there is one.
int enqueue_batch(clx_ctx* ctx, clx_batch* b, cudaStream_t st) {
    if (b->graph) {
        CU(ctx, cudaGraphLaunch(b->graph, st));
        ctx->launches += b->graph_launches;
        return CLX_OK;
    }
    // No graph: two decodes of one batch share its flag words and parameter records, so they must not overlap.
    if (b->ev_idle) CU(ctx, cudaStreamWaitEvent(st, b->ev_idle, 0));
    CU(ctx, launch_batch(b, st, &ctx->launches));
    if (!b->ev_idle) CU(ctx, cudaEventCreateWithFlags(&b->ev_idle, cudaEventDisableTiming));
    CU(ctx, cudaEventRecord(b->ev_idle, st));
    return CLX_OK;
}
}  // namespace

extern "C" {

int clx_batch_decode(clx_ctx* ctx, clx_batch* b, uint32_t stream_index) {
    if (!ctx || !b) return CLX_ERR_INVALID_ARGUMENT;
    cudaStream_t st = ctx->streams[stream_index % ctx->streams.size()];
    b->last_stream = st;
    CU(ctx, cudaEventRecord(b->ev_start, st));
    int rc = enqueue_batch(ctx, b, st);
    if (rc) return rc;
    CU(ctx, cudaEventRecord(b->ev_stop, st));
    return CLX_OK;
}

int clx_batch_sync(clx_ctx* ctx, clx_batch* b) {
    if (!ctx || !b) return CLX_ERR_INVALID_ARGUMENT;
    if (b->last_stream) CU(ctx, cudaStreamSynchronize(b->last_stream));
    return CLX_OK;
}

int clx_batch_last_kernel_ms(clx_ctx* ctx, clx_batch* b, float* ms) {
    if (!ctx || !b || !ms) return CLX_ERR_INVALID_ARGUMENT;
    CU(ctx, cudaEventSynchronize(b->ev_stop));
    CU(ctx, cudaEventElapsedTime(ms, b->ev_start, b->ev_stop));
    return CLX_OK;
}

}  // extern "C"

namespace {
// Per-frame results of the batch's last decode at the caller's frame indices, with the host-side CRC-16 verdicts.
int read_results(clx_ctx* ctx, clx_batch* b, clx_frame_result* results) {
    if (results) {
        std::vector<clx_frame_result> dev(b->n_frames);
        CU(ctx, cudaMemcpy(dev.data(), b->buf.results, b->n_frames * sizeof(clx_frame_result), cudaMemcpyDeviceToHost));
        unpermute(dev.data(), b->order, b->n_frames, results);
        if (!(ctx->flags & CLX_OPT_NO_VERIFY_CRC) && !b->device_crc) {
            std::vector<uint8_t> tmp;
            for (size_t i = 0; i < b->n_frames; i++) {
                if (results[i].status != CLX_OK) continue;
                bool ok;
                const uint32_t consumed = results[i].consumed;
                if (consumed == b->h_len[i]) ok = b->crc_ok[i] != 0;
                else {  // the frame ended before the end of the span it was given: checksum what it did consume
                    if (consumed < 2 || consumed > b->h_len[i]) ok = false;
                    else {
                        tmp.resize(consumed);
                        CU(ctx, cudaMemcpy(tmp.data(), b->buf.bytes + b->h_offset[i], consumed, cudaMemcpyDeviceToHost));
                        const uint16_t stored = (uint16_t)(((uint32_t)tmp[consumed - 2] << 8) | tmp[consumed - 1]);
                        ok = clx_crc16(tmp.data(), consumed - 2) == stored;
                    }
                }
                if (!ok) results[i].status = CLX_ERR_FRAME_CRC_MISMATCH;
            }
        }
    }
    return CLX_OK;
}
}  // namespace

extern "C" {

int clx_batch_read(clx_ctx* ctx, clx_batch* b, int32_t* out, size_t out_elems, clx_frame_result* results) {
    if (!ctx || !b || b->mode != CLX_OUT_PLANAR_I32) return CLX_ERR_INVALID_ARGUMENT;
    return clx_batch_read_to(ctx, b, out, out_elems, results);
}

int clx_batch_read_to(clx_ctx* ctx, clx_batch* b, void* out, size_t out_elems, clx_frame_result* results) {
    if (!ctx || !b) return CLX_ERR_INVALID_ARGUMENT;
    int rc = clx_batch_sync(ctx, b);
    if (rc) return rc;
    if (out)
        CU(ctx, cudaMemcpy(out, clx_batch_device_out(b), std::min(out_elems, b->out_elems) * clx::output_elem_size(b->mode),
                           cudaMemcpyDeviceToHost));
    return read_results(ctx, b, results);
}

void clx_batch_destroy(clx_ctx* ctx, clx_batch* b) {
    (void)ctx;
    if (!b) return;
    b->buf.release();
    for (void* p : b->owned) cudaFree(p);
    clx_batch_destroy(ctx, b->inner);
    if (b->corpus) b->corpus->live--;
    if (b->graph) cudaGraphExecDestroy(b->graph);
    if (b->ev_idle) cudaEventDestroy(b->ev_idle);
    if (b->ev_start) cudaEventDestroy(b->ev_start);
    if (b->ev_stop) cudaEventDestroy(b->ev_stop);
    delete b;
}

// Decodes `steps` batches back to back, step i taking batches[i % n_batches] on internal stream
// i % n_streams, and returns the device time (CUDA events) from the first launch to the last
// completion.  This is the steady-state "many batches in flight" regime of a decode service.
int clx_ctx_run_steps(clx_ctx* ctx, clx_batch** batches, size_t n_batches, uint32_t steps, uint32_t n_streams,
                      float* total_ms) {
    if (!ctx || !batches || n_batches == 0 || !total_ms) return CLX_ERR_INVALID_ARGUMENT;
    CU(ctx, cudaSetDevice(ctx->device));
    n_streams = std::max<uint32_t>(1, std::min<uint32_t>(n_streams, (uint32_t)ctx->streams.size()));
    cudaEvent_t start = nullptr, stop = nullptr;
    std::vector<cudaEvent_t> done(n_streams, nullptr);
    auto body = [&]() -> int {
        CU(ctx, cudaEventCreate(&start));
        CU(ctx, cudaEventCreate(&stop));
        for (auto& e : done) CU(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        cudaStream_t s0 = ctx->streams[0];
        CU(ctx, cudaEventRecord(start, s0));
        for (uint32_t s = 1; s < n_streams; s++) CU(ctx, cudaStreamWaitEvent(ctx->streams[s], start, 0));
        for (uint32_t i = 0; i < steps; i++) {
            clx_batch* b = batches[i % n_batches];
            cudaStream_t st = ctx->streams[i % n_streams];
            b->last_stream = st;
            int rc = enqueue_batch(ctx, b, st);
            if (rc) return rc;
        }
        for (uint32_t s = 1; s < n_streams; s++) {
            CU(ctx, cudaEventRecord(done[s], ctx->streams[s]));
            CU(ctx, cudaStreamWaitEvent(s0, done[s], 0));
        }
        CU(ctx, cudaEventRecord(stop, s0));
        CU(ctx, cudaEventSynchronize(stop));
        CU(ctx, cudaEventElapsedTime(total_ms, start, stop));
        return CLX_OK;
    };
    const int rc = body();
    if (rc != CLX_OK) cudaDeviceSynchronize();  // nothing of this call may still be running when it returns
    if (start) cudaEventDestroy(start);
    if (stop) cudaEventDestroy(stop);
    for (auto& e : done)
        if (e) cudaEventDestroy(e);
    return rc;
}

void* clx_batch_device_out(clx_batch* b) { return b ? (b->mode == CLX_OUT_PLANAR_I32 ? (void*)b->buf.out : b->buf.conv) : nullptr; }
void* clx_batch_device_bytes(clx_batch* b) { return b ? b->buf.bytes : nullptr; }

// Pinned host memory for callers that want true asynchronous copies.
void* clx_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
void clx_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"

// ---------------------------------------------------------------------------------
// device-resident corpora and crop batches (the kernels: clx_crops.cu)
// ---------------------------------------------------------------------------------
namespace {
// Registrations of corpus images' bytes regions (clx_corpus_attach), process-wide: the same range registered twice is
// a CUDA error, so contexts that attach one mapping share one registration, counted, and the last detach drops it.
struct Registry {
    std::mutex m;
    std::map<std::pair<const void*, size_t>, int> refs;
};
Registry& registry() {
    static Registry* r = new Registry();  // (never destroyed: a corpus may outlive static destruction order)
    return *r;
}

cudaError_t register_range(void* p, size_t n) {
    Registry& r = registry();
    std::lock_guard<std::mutex> g(r.m);
    auto it = r.refs.find({p, n});
    if (it != r.refs.end()) {
        it->second++;
        return cudaSuccess;
    }
    const cudaError_t e = cudaHostRegister(p, n, cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e == cudaSuccess) r.refs[{p, n}] = 1;
    else cudaGetLastError();  // (reported here; a later launch check must not see it again)
    return e;
}

void unregister_range(void* p, size_t n) {
    Registry& r = registry();
    std::lock_guard<std::mutex> g(r.m);
    auto it = r.refs.find({p, n});
    if (it == r.refs.end() || --it->second > 0) return;
    r.refs.erase(it);
    cudaHostUnregister(p);
}

void free_corpus(clx_corpus* c) {
    cudaFree(c->d_bytes); cudaFree(c->d_descs); cudaFree(c->d_starts); cudaFree(c->d_file_frames);
    cudaFree(c->d_file_len); cudaFree(c->d_file_ch); cudaFree(c->d_file_tail);
    if (c->attached) unregister_range(c->h_bytes, c->buf_bytes);
    else if (c->h_bytes) cudaFreeHost(c->h_bytes);
    delete c;
}

// Uploads a corpus's frame index: its descriptors (c->descs, the filler frame last), each frame's start, each file's
// frame range (c->file_frames), length, channel count and trailing-bytes verdict `tail`; sets c->channels / max_bps.
cudaError_t upload_index(clx_corpus* c, const std::vector<int32_t>& tail) {
    std::vector<int64_t> starts(c->n_frames), file_len(c->n_files);
    std::vector<uint32_t> file_ch(c->n_files, 0);
    for (size_t i = 0; i < c->n_files; i++) {
        int64_t at = 0;
        for (size_t f = c->file_frames[i]; f < c->file_frames[i + 1]; f++) {
            starts[f] = at;
            at += c->descs[f].block_size;
            c->channels = std::max<uint32_t>(c->channels, c->descs[f].n_channels);
            c->max_bps = std::max<uint32_t>(c->max_bps, c->descs[f].bits_per_sample);
        }
        file_len[i] = at;
        if (c->file_frames[i + 1] > c->file_frames[i]) file_ch[i] = c->descs[c->file_frames[i + 1] - 1].n_channels;
    }
    cudaError_t e = cudaSuccess;
    auto put = [&](auto*& dst, const auto& v) {
        const size_t size = std::max<size_t>(1, v.size()) * sizeof(v[0]);
        if (e == cudaSuccess) e = cudaMalloc((void**)&dst, size);
        if (e == cudaSuccess) c->device_bytes += size;
        if (e == cudaSuccess && !v.empty()) e = cudaMemcpy(dst, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
    };
    put(c->d_descs, c->descs);
    put(c->d_starts, starts);
    put(c->d_file_frames, c->file_frames);
    put(c->d_file_len, file_len);
    put(c->d_file_ch, file_ch);
    put(c->d_file_tail, tail);
    return e;
}
}  // namespace

// The trailing-bytes verdict of a file whose last frame `d` has an unconfirmed end (load()'s check after the last
// frame): decode the frame; if it decodes and ends before byte_len, the frame header status at its end, unless CLX_EOF.
int clx::tail_verdict(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, clx_frame_desc d, int32_t* verdict) {
    *verdict = CLX_OK;
    d.out_offset = 0;
    std::vector<int32_t> pcm((size_t)d.n_channels * d.block_size);
    clx_frame_result res{};
    const int rc = clx_decode_frames(ctx, bytes, nbytes, &d, 1, pcm.data(), pcm.size(), &res);
    if (rc) return rc;
    if (res.status == CLX_OK && res.consumed < d.byte_len) {
        clx_frame_desc next;
        const uint64_t at = d.byte_offset + res.consumed;
        const int st = clx_parse_frame_header(bytes + at, d.byte_offset + d.byte_len - at, &next, 0);
        if (st != CLX_EOF && st != CLX_OK) *verdict = st;
    }
    return CLX_OK;
}

extern "C" {

int clx_corpus_create(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                      const uint32_t* file_frames, size_t n_files, clx_corpus** out) {
    return clx_corpus_create_ex(ctx, bytes, nbytes, descs, n_frames, file_frames, n_files, 0, out);
}

int clx_corpus_create_ex(clx_ctx* ctx, const uint8_t* bytes, size_t nbytes, const clx_frame_desc* descs, size_t n_frames,
                         const uint32_t* file_frames, size_t n_files, uint32_t flags, clx_corpus** out) {
    if (!ctx || !out || !file_frames) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (flags & ~CLX_CORPUS_HOST) return CLX_ERR_INVALID_ARGUMENT;
    const bool host = flags & CLX_CORPUS_HOST;
    if (n_frames >= UINT32_MAX || n_files >= UINT32_MAX || file_frames[n_files] != n_frames) return CLX_ERR_INVALID_ARGUMENT;
    for (size_t i = 0; i < n_files; i++)
        if (file_frames[i + 1] < file_frames[i]) return CLX_ERR_INVALID_ARGUMENT;
    if (!valid_frames(bytes, nbytes, descs, n_frames, nullptr)) return CLX_ERR_INVALID_ARGUMENT;
    // A host corpus gathers a crop's frames as one span from its first frame's start to its last frame's end.
    for (size_t i = 0; host && i < n_files; i++)
        for (size_t f = file_frames[i] + 1; f < file_frames[i + 1]; f++)
            if (descs[f].byte_offset < descs[f - 1].byte_offset ||
                descs[f].byte_offset + descs[f].byte_len < descs[f - 1].byte_offset + descs[f - 1].byte_len)
                return CLX_ERR_INVALID_ARGUMENT;
    CU(ctx, cudaSetDevice(ctx->device));
    std::vector<int32_t> tail(n_files, CLX_OK);
    for (size_t i = 0; i < n_files; i++) {
        for (size_t f = file_frames[i]; f < file_frames[i + 1]; f++)
            if (descs[f].n_channels != descs[file_frames[i]].n_channels) return CLX_ERR_INVALID_ARGUMENT;
        if (file_frames[i + 1] > file_frames[i]) {
            const clx_frame_desc& last = descs[file_frames[i + 1] - 1];
            if (!(last.flags & CLX_FRAME_CRC16_VERIFIED)) {
                const int rc = clx::tail_verdict(ctx, bytes, nbytes, last, &tail[i]);
                if (rc) return rc;
            }
        }
    }
    uint8_t filler[16];
    const size_t filler_len = clx::filler_frame(filler, sizeof filler);
    clx_frame_desc fd;
    const int fst = clx_parse_frame_header(filler, filler_len, &fd, 0);
    if (fst != CLX_OK) return fst;
    fd.byte_offset = nbytes;
    fd.byte_len = (uint32_t)filler_len;
    fd.flags |= CLX_FRAME_CRC16_VERIFIED;
    fd.out_offset = 0;
    clx_corpus* c = new clx_corpus();
    c->n_frames = (uint32_t)n_frames;
    c->n_files = (uint32_t)n_files;
    c->nbytes = nbytes;
    c->file_frames.assign(file_frames, file_frames + n_files + 1);
    c->descs.assign(descs, descs + n_frames);
    c->descs.push_back(fd);
    c->buf_bytes = padded_bytes(nbytes + filler_len);
    cudaError_t e = cudaSuccess;
    if (host) {  // the crop batches stage what they decode; the filler frame is copied from here into each of them
        e = cudaHostAlloc((void**)&c->h_bytes, c->buf_bytes, cudaHostAllocMapped);
        if (e == cudaSuccess) {
            memset(c->h_bytes, 0, c->buf_bytes);
            if (nbytes) memcpy(c->h_bytes, bytes, nbytes);
            memcpy(c->h_bytes + nbytes, filler, filler_len);
            e = cudaHostGetDevicePointer((void**)&c->d_host, c->h_bytes, 0);
        }
    } else {
        e = cudaMalloc((void**)&c->d_bytes, c->buf_bytes);
        if (e == cudaSuccess) c->device_bytes += c->buf_bytes;
        if (e == cudaSuccess) e = cudaMemset(c->d_bytes, 0, c->buf_bytes);
        if (e == cudaSuccess && nbytes) e = cudaMemcpy(c->d_bytes, bytes, nbytes, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(c->d_bytes + nbytes, filler, filler_len, cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess) e = upload_index(c, tail);
    if (e != cudaSuccess) {
        free_corpus(c);
        return cuda_fail(ctx, e, "clx_corpus_create");
    }
    *out = c;
    return CLX_OK;
}

int clx_corpus_attach(clx_ctx* ctx, void* image, size_t image_bytes, clx_corpus** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx::ImageIndex ix;
    if (!ctx || clx::read_image(image, image_bytes, &ix) != CLX_OK) return CLX_ERR_INVALID_ARGUMENT;
    CU(ctx, cudaSetDevice(ctx->device));
    uint8_t* region = static_cast<uint8_t*>(image) + ix.bytes_offset;
    cudaError_t e = register_range(region, ix.bytes_size);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "clx_corpus_attach: cudaHostRegister");
    clx_corpus* c = new clx_corpus();
    c->attached = true;  // from here on free_corpus drops the registration
    c->h_bytes = region;
    c->buf_bytes = ix.bytes_size;
    c->nbytes = ix.nbytes;
    c->n_files = (uint32_t)ix.tail.size();
    c->n_frames = (uint32_t)ix.descs.size() - 1;
    c->descs = std::move(ix.descs);
    c->file_frames = std::move(ix.file_frames);
    e = cudaHostGetDevicePointer((void**)&c->d_host, region, 0);
    if (e == cudaSuccess) e = upload_index(c, ix.tail);
    if (e != cudaSuccess) {
        free_corpus(c);
        return cuda_fail(ctx, e, "clx_corpus_attach");
    }
    *out = c;
    return CLX_OK;
}

int clx_corpus_destroy(clx_ctx* ctx, clx_corpus* corpus) {
    (void)ctx;
    if (!corpus) return CLX_OK;
    if (corpus->live > 0) return CLX_ERR_INVALID_ARGUMENT;
    free_corpus(corpus);
    return CLX_OK;
}

size_t clx_corpus_device_bytes(const clx_corpus* corpus) { return corpus ? corpus->device_bytes : 0; }

}  // extern "C"

namespace {
using Kind = clx_batch::Kind;

// A batch of a corpus kind, counted by the corpus until clx_batch_destroy; a wrapper's `inner` is destroyed with it.
clx_batch* new_batch(Kind kind, clx_corpus* corpus, clx_batch* inner = nullptr) {
    clx_batch* b = new clx_batch();
    b->kind = kind;
    b->corpus = corpus;
    b->inner = inner;
    corpus->live++;
    return b;
}

// A device array of n elements that b owns: uninitialised (device_alloc) or zeroed (device_zeros).
template <typename T>
cudaError_t device_alloc(clx_batch* b, T*& p, size_t n) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, n * sizeof(T));
    if (e == cudaSuccess) b->owned.push_back(q);
    p = static_cast<T*>(q);
    return e;
}
template <typename T>
cudaError_t device_zeros(clx_batch* b, T*& p, size_t n) {
    const cudaError_t e = device_alloc(b, p, n);
    return e == cudaSuccess ? cudaMemset((void*)p, 0, n * sizeof(T)) : e;
}
// A device copy of a host table that b owns (one element at least, so that an empty table is a valid pointer too).
template <typename T>
cudaError_t upload(clx_batch* b, const T*& p, const std::vector<T>& v) {
    T* q = nullptr;
    cudaError_t e = device_alloc(b, q, std::max<size_t>(v.size(), 1));
    p = q;
    if (e == cudaSuccess && !v.empty()) e = cudaMemcpy(q, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
    return e;
}
// A wrapper's float32 output in buf.conv, zeroed, with the slack of DecodeStorage::fit (buf.release() frees it).
cudaError_t alloc_output(clx_batch* b) {
    const size_t bytes = (b->out_elems + 8) * sizeof(float);
    const cudaError_t e = cudaMalloc((void**)&b->buf.conv, bytes);
    return e == cudaSuccess ? cudaMemset(b->buf.conv, 0, bytes) : e;
}

// Crop and packed batches: the corpus and mode they accept; their decode plan (every frame of the corpus, the filler
// frame included) and its planar elements per slot.
bool planned_ok(const clx_ctx* ctx, const clx_corpus* corpus, uint32_t mode) {
    return ctx && corpus && is_channels(mode) && !(mode == CLX_OUT_CHANNELS_F32 && corpus->max_bps > 24);
}
clx::Plan corpus_plan(const clx_ctx* ctx, const clx_corpus* corpus, size_t* slot_elems) {
    const clx::Plan plan = make_plan(ctx, corpus->descs.data(), corpus->descs.size());
    *slot_elems = ((size_t)plan.max_frame_elems + 3) & ~(size_t)3;
    return plan;
}
// The buffers crop and packed batches share, once the kind has set b->ex's sizes and b->staging: the frame bytes (the
// corpus's, or over a host corpus `staging` bytes of staging and then the filler frame), the slots' planar scratch, an
// output of conv_elems elements (trash included), and the planner's per-excerpt buffers.
cudaError_t alloc_planned(clx_ctx* ctx, clx_batch* b, const clx::Plan& plan, uint32_t mode, size_t conv_elems) {
    const clx_corpus* c = b->corpus;
    clx::ExcerptBuffers& eb = b->ex;
    const size_t n = eb.n, staged = b->staging, filler_len = clx::filler_frame(nullptr, 0);
    b->n_frames = eb.n_slots;
    b->plan = plan;
    b->mode = mode;
    b->device_crc = !(ctx->flags & CLX_OPT_NO_VERIFY_CRC);
    if (!c->h_bytes) b->buf.borrow(c->d_bytes, c->buf_bytes);
    cudaError_t e = b->buf.fit({staged + filler_len, eb.n_slots, (size_t)eb.n_slots * eb.slot_elems, mode, conv_elems,
                                true, plan}, false);
    if (e == cudaSuccess && c->h_bytes)
        e = cudaMemcpy(b->buf.bytes + staged, c->h_bytes + c->nbytes, filler_len, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = device_zeros(b, eb.status, n);
    if (e == cudaSuccess) e = device_zeros(b, eb.lengths, n);
    if (e == cudaSuccess) e = device_alloc(b, eb.error, 1);
    if (e == cudaSuccess) e = cudaMemset(eb.error, 0xff, sizeof(unsigned long long));
    if (e == cudaSuccess) e = device_alloc(b, eb.plan, n);
    if (e == cudaSuccess) e = device_alloc(b, eb.scan, n + 1);
    if (e == cudaSuccess) e = device_zeros(b, eb.stage, n);
    if (e == cudaSuccess) e = device_zeros(b, eb.chunks, n + 1);
    return e;
}

// The first half of each corpus batch's create (finish() is the second): a refusal, or CLX_OK with *out the batch and
// *e the first CUDA error of making its buffers.  A wrapper makes its inner batch the same way.
int make_crops(clx_ctx* ctx, clx_corpus* corpus, size_t n_crops, size_t num_frames, uint32_t mode, clx_batch** out,
               cudaError_t* e) {
    if (!planned_ok(ctx, corpus, mode) || n_crops == 0 || num_frames == 0 || n_crops >= (1u << 30))
        return CLX_ERR_INVALID_ARGUMENT;
    const size_t S = clx_crop_frames_bound(corpus->descs.data(), corpus->n_frames, corpus->file_frames.data(),
                                           corpus->n_files, num_frames);
    const size_t C = corpus->channels, rows = n_crops * C;  // (< 2^33: no overflow)
    size_t slot_elems;
    const clx::Plan plan = corpus_plan(ctx, corpus, &slot_elems);
    if (S == 0 || S > UINT32_MAX / n_crops || num_frames > (SIZE_MAX / 4 - 8) / (rows + C)) return CLX_ERR_INVALID_ARGUMENT;
    const size_t slots = n_crops * S;
    if (slots > (SIZE_MAX / 4 - 8) / slot_elems) return CLX_ERR_INVALID_ARGUMENT;
    // Over a host corpus, the batch's own frame bytes: room for n_crops spans of the bytes bound + 15, each rounded up
    // to 16 (the spans are packed from 0 by the planner), then the filler frame.
    size_t span_stride = 0;
    if (corpus->h_bytes) {
        const size_t span = clx_crop_bytes_bound(corpus->descs.data(), corpus->n_frames, corpus->file_frames.data(),
                                                 corpus->n_files, num_frames);
        span_stride = (span + 15 + 15) & ~(size_t)15;
        if (span_stride > (SIZE_MAX / 2) / n_crops) return CLX_ERR_INVALID_ARGUMENT;
    }
    CU(ctx, cudaSetDevice(ctx->device));
    clx_batch* b = *out = new_batch(Kind::Crops, corpus);
    b->staging = n_crops * span_stride;
    b->out_elems = rows * num_frames;
    b->stride = num_frames;
    clx::ExcerptBuffers& eb = b->ex;
    eb.n = (uint32_t)n_crops;
    eb.C = (uint32_t)C;
    eb.n_slots = (uint32_t)slots;
    eb.L = num_frames;
    eb.slot_elems = (uint32_t)slot_elems;
    // the output plus C trash rows for the unused slots
    *e = alloc_planned(ctx, b, plan, mode, (rows + C) * num_frames);
    if (*e == cudaSuccess) *e = device_zeros(b, eb.crop_requests, n_crops);
    return CLX_OK;
}

int make_packed(clx_ctx* ctx, clx_corpus* corpus, size_t max_excerpts, size_t max_samples, uint32_t mode,
                clx_batch** out, cudaError_t* e) {
    if (!planned_ok(ctx, corpus, mode) || max_excerpts == 0 || max_samples == 0 || max_excerpts >= (1u << 30) ||
        max_samples > SIZE_MAX / 16)
        return CLX_ERR_INVALID_ARGUMENT;
    const clx_frame_desc* descs = corpus->descs.data();
    const uint32_t* ff = corpus->file_frames.data();
    const size_t S = clx_packed_frames_bound(descs, corpus->n_frames, ff, corpus->n_files, max_excerpts, max_samples);
    uint32_t largest = 0;  // block size, the filler frame's included (the unused slots decode it into the trash)
    for (const clx_frame_desc& d : corpus->descs) largest = std::max<uint32_t>(largest, d.block_size);
    const size_t T4 = (max_samples + 3) & ~(size_t)3, W = (std::min<size_t>(max_samples, largest) + 3) & ~(size_t)3;
    const size_t C = corpus->channels, stride = T4 + W;
    size_t slot_elems;
    const clx::Plan plan = corpus_plan(ctx, corpus, &slot_elems);
    if (S == 0 || S >= UINT32_MAX || stride > (SIZE_MAX / 4 - 8) / C || S > (SIZE_MAX / 4 - 8) / slot_elems)
        return CLX_ERR_INVALID_ARGUMENT;
    // Over a host corpus, the batch's own frame bytes: the excerpts' spans packed from 0 (at most the bytes bound), then
    // the filler frame.
    size_t staging = 0;
    if (corpus->h_bytes) {
        staging = clx_packed_bytes_bound(descs, corpus->n_frames, ff, corpus->n_files, max_excerpts, max_samples);
        if (staging > SIZE_MAX / 2) return CLX_ERR_INVALID_ARGUMENT;
    }
    CU(ctx, cudaSetDevice(ctx->device));
    clx_batch* b = *out = new_batch(Kind::Packed, corpus);
    b->staging = staging;
    b->out_elems = C * stride;
    b->stride = stride;
    clx::ExcerptBuffers& eb = b->ex;
    eb.n = (uint32_t)max_excerpts;
    eb.C = (uint32_t)C;
    eb.n_slots = (uint32_t)S;
    eb.L = stride;
    eb.T = max_samples;
    eb.slot_elems = (uint32_t)slot_elems;
    // the output with its trash columns, zeroed here: afterwards every call zeroes what it must
    *e = alloc_planned(ctx, b, plan, mode, C * stride);
    if (*e == cudaSuccess) *e = device_zeros(b, eb.packed_requests, max_excerpts);
    if (*e == cudaSuccess) *e = device_zeros(b, eb.count, 1);
    if (*e == cudaSuccess) *e = device_zeros(b, eb.starts, max_excerpts);
    if (*e == cudaSuccess) *e = device_zeros(b, eb.end, 2);
    return CLX_OK;
}

// Resampled crop and packed batches, once the kind has set b->out_elems: the filter of n excerpts of C rows into rows
// of L outputs, with the tables `t`, reading the inner packed batch's source spans.  Status and error word are the
// inner batch's, the lengths at the target rate the batch's own.
cudaError_t fill_resample(clx_batch* b, const clx::ResampleTables& t, size_t n, size_t C, uint64_t L) {
    const clx_batch* inner = b->inner;
    b->mode = CLX_OUT_CHANNELS_F32;
    b->stride = L;
    clx::ExcerptBuffers& eb = b->ex;
    eb.n = (uint32_t)n;
    eb.C = (uint32_t)C;
    eb.L = L;
    eb.status = inner->ex.status;
    eb.error = inner->ex.error;
    clx::ResampleBuffers& rs = b->rs;
    rs.n_crops = (uint32_t)n;
    rs.C = (uint32_t)C;
    rs.L = L;
    rs.tile = t.tile;
    rs.excerpts = const_cast<clx_packed_request*>(inner->ex.packed_requests);
    rs.count = const_cast<uint32_t*>(inner->ex.count);
    rs.starts = inner->ex.starts;
    rs.src = static_cast<const float*>((const void*)inner->buf.conv);
    rs.src_stride = inner->stride;
    cudaError_t e = device_zeros(b, eb.lengths, n);
    if (e == cudaSuccess) e = alloc_output(b);
    if (e == cudaSuccess) e = device_alloc(b, rs.plan, n);
    if (e == cudaSuccess) e = upload(b, rs.file_rate, t.file_rate);
    if (e == cudaSuccess) e = upload(b, rs.rates, t.rates);
    if (e == cudaSuccess) e = upload(b, rs.coefs, t.coefs);
    if (e == cudaSuccess) e = upload(b, rs.k0, t.k0);
    rs.lengths = eb.lengths;
    rs.out = reinterpret_cast<float*>(b->buf.conv);
    return e;
}

int make_resampled_crops(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files, size_t n_crops,
                         size_t num_frames, uint32_t target_rate, clx_batch** out, cudaError_t* e) {
    if (!ctx || !corpus || !file_rates || n_files != corpus->n_files || n_crops == 0 || num_frames == 0 ||
        n_crops >= (1u << 30))
        return CLX_ERR_INVALID_ARGUMENT;
    clx::ResampleTables t;
    if (!clx::resample_tables(file_rates, n_files, target_rate, num_frames, &t)) return CLX_ERR_INVALID_ARGUMENT;
    // The inner packed batch: every crop's source span fits in its round_up_4(bound) columns.
    const size_t C = corpus->channels, rows = n_crops * C;  // (< 2^33: no overflow)
    if (t.bound > (SIZE_MAX / 16) / n_crops || num_frames > (SIZE_MAX / 4 - 8) / rows ||
        (num_frames + t.tile - 1) / t.tile >= (1u << 31))
        return CLX_ERR_INVALID_ARGUMENT;
    clx_batch* inner = nullptr;
    const int rc = make_packed(ctx, corpus, n_crops, n_crops * ((t.bound + 3) & ~(size_t)3), CLX_OUT_CHANNELS_F32,
                               &inner, e);
    if (rc != CLX_OK) return rc;
    clx_batch* b = *out = new_batch(Kind::ResampledCrops, corpus, inner);
    b->out_elems = rows * num_frames;
    if (*e == cudaSuccess) *e = fill_resample(b, t, n_crops, C, num_frames);
    if (*e == cudaSuccess) *e = device_zeros(b, b->ex.crop_requests, n_crops);
    return CLX_OK;
}

int make_resampled_packed(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                          size_t max_excerpts, size_t max_samples, uint32_t target_rate, clx_batch** out,
                          cudaError_t* e) {
    if (!ctx || !corpus || !file_rates || n_files != corpus->n_files || max_excerpts == 0 || max_samples == 0 ||
        max_excerpts >= (1u << 30) || max_samples > SIZE_MAX / 16)
        return CLX_ERR_INVALID_ARGUMENT;
    clx::ResampleTables t;
    if (!clx::resample_tables(file_rates, n_files, target_rate, max_samples, &t)) return CLX_ERR_INVALID_ARGUMENT;
    // The inner packed batch: the source spans of any excerpts that fit in T columns at R fit in its columns.
    const size_t src_cols = clx::resample_packed_bound(t, max_excerpts, max_samples);
    const size_t C = corpus->channels, stride = (max_samples + 3) & ~(size_t)3;
    if (src_cols == SIZE_MAX || stride > (SIZE_MAX / 4 - 8) / C || (stride + t.tile - 1) / t.tile >= (1u << 31))
        return CLX_ERR_INVALID_ARGUMENT;
    clx_batch* inner = nullptr;
    const int rc = make_packed(ctx, corpus, max_excerpts, src_cols, CLX_OUT_CHANNELS_F32, &inner, e);
    if (rc != CLX_OK) return rc;
    clx_batch* b = *out = new_batch(Kind::ResampledPacked, corpus, inner);
    b->out_elems = C * stride;
    b->ex.T = max_samples;
    if (*e == cudaSuccess) *e = fill_resample(b, t, max_excerpts, C, stride);
    if (*e == cudaSuccess) *e = device_zeros(b, b->ex.packed_requests, max_excerpts);
    if (*e == cudaSuccess) *e = device_zeros(b, b->ex.count, 1);
    if (*e == cudaSuccess) *e = device_zeros(b, b->ex.starts, max_excerpts);
    return CLX_OK;
}

// Mel crop and packed batches: the features of `rows` rows of F frames, `tiles` tiles of frames per row, of the inner
// batch's output, with the parameters `p` and the tables `t`.  Requests, status, lengths and error word are the inner
// batch's.
cudaError_t fill_mel(clx_batch* b, const clx_mel_params* p, const clx::MelTables& t, uint64_t F, size_t rows,
                     uint64_t tiles) {
    const clx_batch* inner = b->inner;
    b->ex = inner->ex;
    b->mode = CLX_OUT_CHANNELS_F32;
    b->stride = F;
    b->out_elems = rows * p->n_mels * F;
    clx::MelBuffers& mb = b->mel;
    mb.src = reinterpret_cast<const float*>(inner->buf.conv);
    mb.L = inner->stride;
    mb.F = F;
    mb.rows = (uint32_t)rows;
    mb.tiles = (uint32_t)tiles;
    mb.n_fft = p->n_fft;
    mb.hop = p->hop_length;
    mb.n_mels = p->n_mels;
    mb.tile = t.tile;
    mb.flags = p->flags;
    mb.log_floor = p->log_floor;
    mb.log_of_floor = (p->flags & CLX_MEL_LOG) ? (float)std::log((double)p->log_floor) : 0.f;
    b->mel_smem = t.smem;
    cudaError_t e = clx::mel_init();
    if (e == cudaSuccess) e = alloc_output(b);
    if (e == cudaSuccess) e = upload(b, mb.tw, t.tw);
    if (e == cudaSuccess) e = upload(b, mb.window, t.window);
    if (e == cudaSuccess) e = upload(b, mb.bands, t.bands);
    if (e == cudaSuccess) e = upload(b, mb.weights, t.weights);
    mb.out = reinterpret_cast<float*>(b->buf.conv);
    clx::MelNorm& mn = b->mel_norm;  // the layout fields; the caller sets the lengths or the packed plan
    mn.out = mb.out;
    mn.F = F;
    mn.C = b->corpus->channels;
    mn.n_mels = p->n_mels;
    mn.hop = p->hop_length;
    mn.flags = p->flags & (CLX_MEL_NORM_PER_FEATURE | CLX_MEL_NORM_WHISPER);
    return e;
}

int make_mel_crops(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files, size_t n_crops,
                   size_t num_frames, uint32_t target_rate, const clx_mel_params* params, const float* window,
                   const float* fbank, clx_batch** out, cudaError_t* e) {
    if (!ctx || !corpus || n_crops == 0 || n_crops >= (1u << 30)) return CLX_ERR_INVALID_ARGUMENT;
    clx::MelTables t;
    if (!clx::mel_tables(params, window, fbank, &t)) return CLX_ERR_INVALID_ARGUMENT;
    const bool whisper = params->flags & CLX_MEL_NORM_WHISPER;
    uint64_t F = clx::mel_frame_count(num_frames, params->n_fft, params->hop_length, params->flags & CLX_MEL_CENTER);
    if (F == 0) return CLX_ERR_INVALID_ARGUMENT;  // a row too short for a frame, or for the reflect pad
    if (whisper && F-- < 2) return CLX_ERR_INVALID_ARGUMENT;  // Whisper drops the last frame: it needs two
    const size_t C = corpus->channels, rows = n_crops * C;  // (< 2^33: no overflow)
    const uint64_t tiles = (F + t.tile - 1) / t.tile;
    if (F > (SIZE_MAX / 4 - 8) / (rows * params->n_mels) || tiles >= (1u << 31) / rows) return CLX_ERR_INVALID_ARGUMENT;
    if ((params->flags & CLX_MEL_NORM_PER_FEATURE) && rows * params->n_mels >= (1u << 31))
        return CLX_ERR_INVALID_ARGUMENT;  // mel_norm_kernel numbers its (row, mel) segments in 32 bits
    clx_batch* inner = nullptr;
    const int rc = target_rate ? make_resampled_crops(ctx, corpus, file_rates, n_files, n_crops, num_frames,
                                                      target_rate, &inner, e)
                               : make_crops(ctx, corpus, n_crops, num_frames, CLX_OUT_CHANNELS_F32, &inner, e);
    if (rc != CLX_OK) return rc;
    clx_batch* b = *out = new_batch(Kind::MelCrops, corpus, inner);
    if (*e == cudaSuccess) *e = fill_mel(b, params, t, F, rows, tiles);
    b->mel_norm.lengths = b->ex.lengths;
    b->mel_norm.n = (uint32_t)n_crops;
    return CLX_OK;
}

int make_mel_packed(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files, size_t max_excerpts,
                    size_t max_samples, uint32_t target_rate, const clx_mel_params* params, const float* window,
                    const float* fbank, clx_batch** out, cudaError_t* e) {
    if (!ctx || !corpus || max_excerpts == 0 || max_excerpts >= (1u << 30) || max_samples == 0)
        return CLX_ERR_INVALID_ARGUMENT;
    clx::MelTables t;
    if (!clx::mel_tables(params, window, fbank, &t) || (params->flags & CLX_MEL_NORM_WHISPER))
        return CLX_ERR_INVALID_ARGUMENT;  // (Whisper's input is a fixed window: crops only)
    const size_t F = clx::mel_packed_frames(params, max_excerpts, max_samples), C = corpus->channels;
    const uint64_t tiles = std::max<uint64_t>(1, (F + t.tile - 1) / t.tile);  // (one CTA per row when F is 0)
    if (F == SIZE_MAX || F > (SIZE_MAX / 4 - 8) / (C * params->n_mels) || tiles >= (1u << 31) / C)
        return CLX_ERR_INVALID_ARGUMENT;
    if ((params->flags & CLX_MEL_NORM_PER_FEATURE) && max_excerpts * C * params->n_mels >= (1u << 31))
        return CLX_ERR_INVALID_ARGUMENT;  // mel_norm_kernel numbers its (excerpt, row, mel) segments in 32 bits
    clx_batch* inner = nullptr;
    const int rc = target_rate ? make_resampled_packed(ctx, corpus, file_rates, n_files, max_excerpts, max_samples,
                                                       target_rate, &inner, e)
                               : make_packed(ctx, corpus, max_excerpts, max_samples, CLX_OUT_CHANNELS_F32, &inner, e);
    if (rc != CLX_OK) return rc;
    clx_batch* b = *out = new_batch(Kind::MelPacked, corpus, inner);
    clx::MelPacked& mp = b->mel_packed;
    mp.count = inner->ex.count;
    mp.lengths = inner->ex.lengths;
    mp.src_starts = inner->ex.starts;
    mp.n = (uint32_t)max_excerpts;
    if (*e == cudaSuccess) *e = fill_mel(b, params, t, F, C, tiles);  // b->ex: the inner batch's, but for the starts
    if (*e == cudaSuccess) *e = device_zeros(b, b->ex.starts, max_excerpts);
    if (*e == cudaSuccess) *e = device_zeros(b, mp.frames, max_excerpts);
    mp.starts = b->ex.starts;
    b->mel_norm.count = mp.count;
    b->mel_norm.starts = mp.starts;
    b->mel_norm.frames = mp.frames;
    b->mel_norm.n = mp.n;
    return CLX_OK;
}

bool corpus_kind(const clx_batch* b) { return b && b->kind != Kind::Frames; }
bool packed_kind(const clx_batch* b) {
    return b && (b->kind == Kind::Packed || b->kind == Kind::ResampledPacked || b->kind == Kind::MelPacked);
}
}  // namespace

extern "C" {

int clx_batch_create_crops(clx_ctx* ctx, clx_corpus* corpus, size_t n_crops, size_t num_frames, uint32_t mode,
                           clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_batch* b = nullptr;
    cudaError_t e = cudaSuccess;
    const int rc = make_crops(ctx, corpus, n_crops, num_frames, mode, &b, &e);
    return rc ? rc : finish(ctx, b, e, "clx_batch_create_crops", out);
}

void* clx_batch_crop_requests(clx_batch* b) { return corpus_kind(b) ? (void*)b->ex.crop_requests : nullptr; }
void* clx_batch_crop_status(clx_batch* b) { return corpus_kind(b) ? (void*)b->ex.status : nullptr; }
void* clx_batch_crop_lengths(clx_batch* b) { return corpus_kind(b) ? (void*)b->ex.lengths : nullptr; }
void* clx_batch_crop_error(clx_batch* b) { return corpus_kind(b) ? (void*)b->ex.error : nullptr; }

int clx_batch_create_packed(clx_ctx* ctx, clx_corpus* corpus, size_t max_excerpts, size_t max_samples, uint32_t mode,
                            clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_batch* b = nullptr;
    cudaError_t e = cudaSuccess;
    const int rc = make_packed(ctx, corpus, max_excerpts, max_samples, mode, &b, &e);
    return rc ? rc : finish(ctx, b, e, "clx_batch_create_packed", out);
}

void* clx_batch_packed_requests(clx_batch* b) { return packed_kind(b) ? (void*)b->ex.packed_requests : nullptr; }
void* clx_batch_packed_count(clx_batch* b) { return packed_kind(b) ? (void*)b->ex.count : nullptr; }
void* clx_batch_packed_starts(clx_batch* b) { return packed_kind(b) ? (void*)b->ex.starts : nullptr; }
size_t clx_batch_packed_stride(clx_batch* b) { return packed_kind(b) ? b->stride : 0; }

int clx_batch_create_resampled_crops(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                                     size_t n_crops, size_t num_frames, uint32_t target_rate, clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_batch* b = nullptr;
    cudaError_t e = cudaSuccess;
    const int rc = make_resampled_crops(ctx, corpus, file_rates, n_files, n_crops, num_frames, target_rate, &b, &e);
    return rc ? rc : finish(ctx, b, e, "clx_batch_create_resampled_crops", out);
}

int clx_batch_create_resampled_packed(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                                      size_t max_excerpts, size_t max_samples, uint32_t target_rate, clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_batch* b = nullptr;
    cudaError_t e = cudaSuccess;
    const int rc = make_resampled_packed(ctx, corpus, file_rates, n_files, max_excerpts, max_samples, target_rate, &b,
                                         &e);
    return rc ? rc : finish(ctx, b, e, "clx_batch_create_resampled_packed", out);
}

int clx_batch_create_mel_crops(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                               size_t n_crops, size_t num_frames, uint32_t target_rate, const clx_mel_params* params,
                               const float* window, const float* fbank, clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_batch* b = nullptr;
    cudaError_t e = cudaSuccess;
    const int rc = make_mel_crops(ctx, corpus, file_rates, n_files, n_crops, num_frames, target_rate, params, window,
                                  fbank, &b, &e);
    return rc ? rc : finish(ctx, b, e, "clx_batch_create_mel_crops", out);
}

int clx_batch_create_mel_packed(clx_ctx* ctx, clx_corpus* corpus, const uint32_t* file_rates, size_t n_files,
                                size_t max_excerpts, size_t max_samples, uint32_t target_rate,
                                const clx_mel_params* params, const float* window, const float* fbank,
                                clx_batch** out) {
    if (!out) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_batch* b = nullptr;
    cudaError_t e = cudaSuccess;
    const int rc = make_mel_packed(ctx, corpus, file_rates, n_files, max_excerpts, max_samples, target_rate, params,
                                   window, fbank, &b, &e);
    return rc ? rc : finish(ctx, b, e, "clx_batch_create_mel_packed", out);
}

void* clx_batch_mel_frames(clx_batch* b) { return b && b->kind == Kind::MelPacked ? (void*)b->mel_packed.frames : nullptr; }

}  // extern "C"

// ---------------------------------------------------------------------------------
// reader facade: claxon::FrameReader / FlacReader::blocks() over the batched device path
// ---------------------------------------------------------------------------------
struct clx_reader {
    clx_ctx* ctx = nullptr;
    const uint8_t* bytes = nullptr;
    size_t n = 0;
    uint64_t pos = 0;
    bool have_si = false;
    clx_streaminfo si{};
    std::vector<clx_frame_desc> descs;
    std::vector<clx_frame_result> results;
    // frames demuxed ahead by clx_reader_plan_batch / clx_reader_next_batch, valid while pos == plan_pos
    size_t plan_n = 0, plan_max = 0;
    uint64_t plan_pos = ~0ull, plan_elems = 0;
    int plan_stop = CLX_OK;
};

namespace {
// Upper bound on the bytes a sane encoder spends on a frame: verbatim coding plus slack.
size_t sane_frame_bound(const clx_frame_desc& d) {
    const size_t per_ch = ((size_t)d.block_size * (d.bits_per_sample + 2u)) / 8 + 256;
    return (size_t)d.header_len + (size_t)d.n_channels * per_ch + 2;
}
uint64_t block_time(const clx_frame_desc& d) {  // src/frame.rs:771-774
    return (d.flags & CLX_FRAME_VARIABLE_BLOCKING) ? d.number : (uint64_t)d.block_size * d.number;
}
}  // namespace

extern "C" {

int clx_reader_open_frames(clx_ctx* ctx, const uint8_t* bytes, size_t n, clx_reader** out) {
    if (!ctx || !out || (!bytes && n)) return CLX_ERR_INVALID_ARGUMENT;
    clx_reader* r = new clx_reader();
    r->ctx = ctx;
    r->bytes = bytes;
    r->n = n;
    *out = r;
    return CLX_OK;
}

int clx_reader_open_flac(clx_ctx* ctx, const uint8_t* bytes, size_t n, clx_reader** out) {
    if (!ctx || !out || (!bytes && n)) return CLX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    clx_streaminfo si;
    uint64_t first = 0;
    int st = clx_open_stream(bytes, n, &si, &first);
    if (st) return st;
    clx_reader* r = new clx_reader();
    r->ctx = ctx;
    r->bytes = bytes;
    r->n = n;
    r->pos = first;
    r->have_si = true;
    r->si = si;
    *out = r;
    return CLX_OK;
}

int clx_reader_streaminfo(const clx_reader* r, clx_streaminfo* si) {
    if (!r || !si || !r->have_si) return CLX_ERR_INVALID_ARGUMENT;
    *si = r->si;
    return CLX_OK;
}

uint64_t clx_reader_position(const clx_reader* r) { return r ? r->pos : 0; }
void clx_reader_close(clx_reader* r) { delete r; }

int clx_reader_next(clx_reader* r, int32_t* buffer, size_t capacity, uint32_t* block_size, uint32_t* channels,
                    uint64_t* time) {
    if (!r) return CLX_ERR_INVALID_ARGUMENT;
    if (r->pos > r->n) return CLX_EOF;
    clx_frame_desc d;
    const size_t avail = r->n - r->pos;
    int st = clx_parse_frame_header(r->bytes + r->pos, avail, &d, r->ctx->flags);
    if (st) return st;  // CLX_EOF == Ok(None)
    if (block_size) *block_size = d.block_size;
    if (channels) *channels = d.n_channels;
    const size_t elems = (size_t)d.n_channels * d.block_size;
    if (capacity < elems || !buffer) return CLX_ERR_INVALID_ARGUMENT;  // ensure_buffer_len is the caller's job
    d.byte_offset = r->pos;
    d.out_offset = 0;
    clx_frame_result res{};
    // A frame does not carry its length; give the device a generous window and widen it to the
    // rest of the stream in the (pathological) case the frame turns out to be longer.
    size_t window = std::min(avail, sane_frame_bound(d));
    for (;;) {
        d.byte_len = (uint32_t)std::min<size_t>(window, (size_t)1 << 28);
        st = clx_decode_frames(r->ctx, r->bytes, r->n, &d, 1, buffer, capacity, &res);
        if (st) return st;
        if (res.status == CLX_ERR_IO_UNEXPECTED_EOF && window < avail) { window = avail; continue; }
        break;
    }
    if (res.status != CLX_OK) return res.status;
    r->pos += res.consumed;
    if (time) *time = block_time(d);
    return CLX_OK;
}

}  // extern "C"

namespace {
// Demuxes up to max_frames frames ahead of the reader's position (once per position).
void plan(clx_reader* r, size_t max_frames) {
    if (r->plan_pos == r->pos && r->plan_max == max_frames) return;
    r->descs.resize(max_frames);
    uint64_t next = r->pos, total = 0;
    int stop = CLX_OK;
    size_t n = 0;
    if (r->pos > r->n) stop = CLX_EOF;
    else n = clx_demux_frames(r->bytes, r->n, r->pos, r->descs.data(), max_frames, &next, &total, &stop, r->ctx->flags);
    r->plan_n = n; r->plan_max = max_frames; r->plan_pos = r->pos; r->plan_elems = total; r->plan_stop = stop;
}
}  // namespace

extern "C" {

int clx_reader_plan_batch(clx_reader* r, size_t max_frames, size_t* n_frames, uint64_t* out_elems) {
    if (!r || !n_frames || !out_elems) return CLX_ERR_INVALID_ARGUMENT;
    *n_frames = 0;
    *out_elems = 0;
    if (max_frames == 0) return CLX_OK;
    plan(r, max_frames);
    if (r->plan_n == 0) return r->plan_stop;  // header-level error or CLX_EOF
    *n_frames = r->plan_n;
    *out_elems = r->plan_elems;
    return CLX_OK;
}

int clx_reader_next_batch(clx_reader* r, size_t max_frames, int32_t* buffer, size_t capacity, clx_frame_desc* descs,
                          size_t* n_decoded) {
    if (!r || !n_decoded || !descs) return CLX_ERR_INVALID_ARGUMENT;
    *n_decoded = 0;
    if (max_frames == 0) return CLX_OK;
    plan(r, max_frames);
    size_t n = r->plan_n;
    if (n == 0) return r->plan_stop;  // header-level error or CLX_EOF
    // fit the caller's buffer
    while (n > 0) {
        const clx_frame_desc& last = r->descs[n - 1];
        if (last.out_offset + (uint64_t)last.n_channels * last.block_size <= capacity) break;
        n--;
    }
    if (n == 0 || !buffer) return CLX_ERR_INVALID_ARGUMENT;  // not even the first frame fits: see clx_reader_plan_batch
    r->results.resize(n);
    int st = clx_decode_frames(r->ctx, r->bytes, r->n, r->descs.data(), n, buffer, capacity, r->results.data());
    if (st) return st;
    size_t good = 0;
    while (good < n && r->results[good].status == CLX_OK) good++;
    if (good == 0) return r->results[0].status;  // the very first frame failed
    for (size_t i = 0; i < good; i++) {
        descs[i] = r->descs[i];
        descs[i].byte_len = r->results[i].consumed;
        descs[i].number = block_time(r->descs[i]);  // Block::time()
    }
    const clx_frame_desc& lastd = r->descs[good - 1];
    r->pos = lastd.byte_offset + r->results[good - 1].consumed;
    *n_decoded = good;
    return CLX_OK;
}

}  // extern "C"

#ifdef CLX_EXPERIMENT
// Measurement builds only (libclaxon_b200_exp.so, tools/exp_*.py): choose which passes of the throughput path a
// batch's graph contains, and rebuild a batch's graph after changing the choice.
extern "C" void clx_exp_set_which(int which) { clx::g_exp_which = which; }
extern "C" void clx_exp_set_dyn_smem(int bytes) { clx::g_exp_dyn_smem = bytes; }
extern "C" int clx_exp_rebuild_graph(clx_ctx* ctx, clx_batch* b) {
    if (!ctx || !b) return CLX_ERR_INVALID_ARGUMENT;
    cudaDeviceSynchronize();
    if (b->graph) { cudaGraphExecDestroy(b->graph); b->graph = nullptr; }
    build_graph(ctx, b);
    return b->graph ? CLX_OK : CLX_ERR_CUDA;
}
#endif
