// claxon_b200.hpp — header-only C++ facade over the C ABI (include/claxon_b200.h) that mirrors the
// names and semantics of claxon's public Rust API for the per-frame decode path:
//
//   claxon::FlacReader::{open,new_,streaminfo,blocks}      reference src/lib.rs:217-470
//   claxon::FrameReader::{read_next_or_eof,into_inner}     reference src/frame.rs:650-785
//   claxon::Block::{time,len,duration,channels,channel,sample,into_buffer}  src/frame.rs:402-529
//   claxon::Error {IoError, FormatError, Unsupported}      reference src/error.rs:18-45
//
// All decoding happens in libclaxon_b200.so (CUDA, sm_90a).  Nothing here decodes on the CPU.
#ifndef CLAXON_B200_HPP
#define CLAXON_B200_HPP

#include <cstdint>
#include <cstring>
#include <fstream>
#include <iterator>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "claxon_b200.h"

namespace claxon {

// claxon::Error: compared by variant + message (src/error.rs:34-45); IoError never compares equal.
class Error : public std::runtime_error {
public:
    enum Kind { IoError = CLX_KIND_IO, FormatError = CLX_KIND_FORMAT, Unsupported = CLX_KIND_UNSUPPORTED,
                Library = CLX_KIND_LIBRARY };
    explicit Error(int status) : std::runtime_error(clx_status_str(status)), status_(status) {}
    int status() const { return status_; }
    Kind kind() const { return static_cast<Kind>(clx_status_kind(status_)); }
    bool operator==(const Error& o) const {
        if (kind() == IoError || o.kind() == IoError) return false;
        return kind() == o.kind() && std::strcmp(what(), o.what()) == 0;
    }
private:
    int status_;
};

// Owns a clx_ctx (one per thread / GPU).
class Context {
public:
    explicit Context(int device = 0, bool verify_crc = true) {
        clx_options o{device, verify_crc ? 0u : CLX_OPT_NO_VERIFY_CRC, 0, 0};
        int st = clx_ctx_create(&o, &ctx_);
        if (st) throw Error(st);
    }
    ~Context() { clx_ctx_destroy(ctx_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    clx_ctx* get() const { return ctx_; }
private:
    clx_ctx* ctx_ = nullptr;
};

// claxon::frame::Block — planar samples, channel-major (src/frame.rs:402-411).
class Block {
public:
    Block() = default;  // Block::empty()
    Block(uint64_t time, uint32_t block_size, std::vector<int32_t> buffer)
        : time_(time), bs_(block_size), channels_(block_size ? uint32_t(buffer.size() / block_size) : 0),
          buffer_(std::move(buffer)) {}
    static Block empty() { return Block(); }
    uint64_t time() const { return time_; }
    uint32_t len() const { return bs_ * channels_; }
    uint32_t duration() const { return bs_; }
    uint32_t channels() const { return channels_; }
    const int32_t* channel(uint32_t ch) const {
        if (ch >= channels_) throw std::out_of_range("channel");  // the reference panics
        return buffer_.data() + size_t(ch) * bs_;
    }
    int32_t sample(uint32_t ch, uint32_t i) const { return buffer_.at(size_t(ch) * bs_ + i); }
    std::vector<int32_t> into_buffer() && { return std::move(buffer_); }
private:
    uint64_t time_ = 0;
    uint32_t bs_ = 0, channels_ = 0;
    std::vector<int32_t> buffer_;
};

// claxon::frame::FrameReader over an in-memory byte span positioned at a frame header.
class FrameReader {
public:
    FrameReader(Context& ctx, const uint8_t* bytes, size_t n) : bytes_(bytes), n_(n) {
        int st = clx_reader_open_frames(ctx.get(), bytes, n, &r_);
        if (st) throw Error(st);
    }
    FrameReader(FrameReader&& o) noexcept : r_(o.r_), bytes_(o.bytes_), n_(o.n_) { o.r_ = nullptr; }
    ~FrameReader() { clx_reader_close(r_); }
    // read_next_or_eof(buffer) -> Result<Option<Block>>: nullopt == Ok(None); throws Error on Err.
    // The buffer is moved in and comes back inside the Block (recycle with into_buffer()).
    std::optional<Block> read_next_or_eof(std::vector<int32_t> buffer) {
        clx_frame_desc d;
        const uint64_t pos = clx_reader_position(r_);
        int st = clx_parse_frame_header(bytes_ + pos, n_ - pos, &d, 0);
        if (st == CLX_EOF) return std::nullopt;
        if (st != CLX_OK && st != CLX_ERR_HEADER_CRC_MISMATCH) throw Error(st);
        buffer.resize(size_t(d.n_channels) * d.block_size);  // ensure_buffer_len (src/frame.rs:616-637)
        uint32_t bs = 0, ch = 0;
        uint64_t time = 0;
        st = clx_reader_next(r_, buffer.data(), buffer.size(), &bs, &ch, &time);
        if (st == CLX_EOF) return std::nullopt;
        if (st) throw Error(st);
        return Block(time, bs, std::move(buffer));
    }
    // Batched extension: up to max_frames frames in one device pass.
    std::vector<Block> read_batch(size_t max_frames) {
        size_t planned = 0;
        uint64_t need = 0;
        int st = clx_reader_plan_batch(r_, max_frames, &planned, &need);  // demux ahead: exact buffer size
        if (st == CLX_EOF) return {};
        if (st) throw Error(st);
        std::vector<clx_frame_desc> descs(max_frames);
        std::vector<int32_t> pcm(size_t(need) + 4);
        size_t n = 0;
        st = clx_reader_next_batch(r_, max_frames, pcm.data(), pcm.size(), descs.data(), &n);
        if (st == CLX_EOF) return {};
        if (st) throw Error(st);
        std::vector<Block> out;
        for (size_t i = 0; i < n; i++) {
            const size_t cnt = size_t(descs[i].n_channels) * descs[i].block_size;
            out.emplace_back(descs[i].number, descs[i].block_size,
                             std::vector<int32_t>(pcm.begin() + descs[i].out_offset,
                                                  pcm.begin() + descs[i].out_offset + cnt));
        }
        return out;
    }
protected:
    friend class FlacReader;
    FrameReader() = default;
    clx_reader* r_ = nullptr;
    const uint8_t* bytes_ = nullptr;
    size_t n_ = 0;
};

// claxon::FlacReader for in-memory streams / files.
class FlacReader {
public:
    static FlacReader open(Context& ctx, const std::string& path) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw std::runtime_error("cannot open " + path);
        std::vector<uint8_t> data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        return FlacReader(ctx, std::move(data));
    }
    FlacReader(Context& ctx, std::vector<uint8_t> data) : data_(std::move(data)) {
        frames_.bytes_ = data_.data();
        frames_.n_ = data_.size();
        int st = clx_reader_open_flac(ctx.get(), data_.data(), data_.size(), &frames_.r_);
        if (st) throw Error(st);
        clx_reader_streaminfo(frames_.r_, &si_);
    }
    const clx_streaminfo& streaminfo() const { return si_; }
    FrameReader& blocks() { return frames_; }
private:
    std::vector<uint8_t> data_;
    FrameReader frames_;
    clx_streaminfo si_{};
};

}  // namespace claxon
#endif
