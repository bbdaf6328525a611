// clx_corpus_image.cpp — corpus images (include/claxon_b200.h, "Shared host corpora"): their layout, the writer and the
// validator.  A host corpus's frame index and bytes in one file that every process of a machine maps; clx_corpus_attach
// (clx_api.cu) registers the bytes region of a checked image and uploads the index read_image() copied out of it.
//
// The image is external input: nothing here trusts a field of it before checking it, and every read is bounded by
// image_bytes.  Only host code; the check needs no context and no device.
#include <stdint.h>
#include <string.h>

#include <atomic>
#include <vector>

#include "claxon_b200.h"
#include "clx_internal.h"

static_assert(sizeof(clx_image_header) == 96, "clx_image_header layout");
static_assert(sizeof(clx_image_file) == 88, "clx_image_file layout");
static_assert(sizeof(clx_frame_desc) == 40, "clx_frame_desc layout");
static_assert(sizeof(clx_streaminfo) == 56, "clx_streaminfo layout");

namespace {
constexpr uint64_t FILES_OFFSET = 128;
constexpr size_t INFO_PAD = offsetof(clx_streaminfo, samples) - 4;  // the 4 padding bytes after bits_per_sample

uint64_t round_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

// The section offsets and sizes an image of these counts has; false for counts the layout refuses.
struct Layout {
    uint64_t files_offset, files_bytes, descs_offset, descs_bytes, bytes_offset, bytes_size, total;
};
bool layout(uint64_t n_files, uint64_t n_frames, uint64_t nbytes, Layout* l) {
    if (n_files >= UINT32_MAX || n_frames >= UINT32_MAX || nbytes > (UINT64_MAX >> 2)) return false;
    l->files_offset = FILES_OFFSET;
    l->files_bytes = n_files * sizeof(clx_image_file);
    l->descs_offset = round_up(l->files_offset + l->files_bytes, 64);
    l->descs_bytes = (n_frames + 1) * sizeof(clx_frame_desc);
    l->bytes_offset = round_up(l->descs_offset + l->descs_bytes, CLX_IMAGE_ALIGN);
    l->bytes_size = clx::padded_bytes(nbytes + clx::filler_frame(nullptr, 0));
    l->total = l->bytes_offset + l->bytes_size;
    return l->total <= SIZE_MAX;
}

// The filler frame's bytes and its descriptor at byte_offset `nbytes`, exactly as clx_corpus_create_ex builds them.
size_t filler(uint64_t nbytes, uint8_t* bytes, clx_frame_desc* fd) {
    const size_t len = clx::filler_frame(bytes, 16);
    memset(fd, 0, sizeof *fd);
    if (clx_parse_frame_header(bytes, len, fd, 0) != CLX_OK) return 0;
    fd->byte_offset = nbytes;
    fd->byte_len = (uint32_t)len;
    fd->flags |= CLX_FRAME_CRC16_VERIFIED;
    fd->out_offset = 0;
    return len;
}

bool all_zero(const uint8_t* p, uint64_t n) {
    for (uint64_t i = 0; i < n; i++)
        if (p[i]) return false;
    return true;
}

// What clx_corpus_create_ex(..., CLX_CORPUS_HOST) requires of one file's frames beyond their byte range: byte order
// (a crop's frames are gathered as one span) and one channel count.
bool file_frames_ok(const clx_frame_desc* d, size_t n) {
    for (size_t f = 1; f < n; f++)
        if (d[f].byte_offset < d[f - 1].byte_offset ||
            d[f].byte_offset + d[f].byte_len < d[f - 1].byte_offset + d[f - 1].byte_len || d[f].n_channels != d[0].n_channels)
            return false;
    return true;
}

// The frame ranges are monotone and end at n_frames, and each file's first frame lies in it; then the bytes the region
// takes for the files (each from its first frame to its end).
bool region_bytes(const size_t* file_nbytes, const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames,
                  size_t n_files, uint64_t* nbytes) {
    if (!file_frames || (n_files && !file_nbytes) || (n_frames && !descs) || n_files >= UINT32_MAX ||
        n_frames >= UINT32_MAX || file_frames[0] != 0 || file_frames[n_files] != n_frames)
        return false;
    uint64_t sum = 0;
    for (size_t i = 0; i < n_files; i++) {
        if (file_frames[i + 1] < file_frames[i]) return false;
        if (file_frames[i + 1] == file_frames[i]) continue;
        const uint64_t first = descs[file_frames[i]].byte_offset;
        if (first > file_nbytes[i] || file_nbytes[i] - first > (UINT64_MAX >> 2) - sum) return false;
        sum += file_nbytes[i] - first;
    }
    *nbytes = sum;
    return true;
}
}  // namespace

namespace clx {

int read_image(const void* image, size_t image_bytes, ImageIndex* ix) {
    const int BAD = CLX_ERR_INVALID_ARGUMENT;
    const uint8_t* p = static_cast<const uint8_t*>(image);
    if (!p || image_bytes < sizeof(clx_image_header)) return BAD;
    clx_image_header h;
    memcpy(&h, p, sizeof h);
    Layout l;
    if (h.magic != CLX_IMAGE_MAGIC || h.version != CLX_IMAGE_VERSION || h.header_bytes != sizeof h ||
        !layout(h.n_files, h.n_frames, h.nbytes, &l))
        return BAD;
    if (h.files_offset != l.files_offset || h.files_bytes != l.files_bytes || h.descs_offset != l.descs_offset ||
        h.descs_bytes != l.descs_bytes || h.bytes_offset != l.bytes_offset || h.bytes_size != l.bytes_size ||
        h.total_bytes != l.total || image_bytes != l.total)
        return BAD;
    // (from here on every section lies inside the image)
    if (!all_zero(p + sizeof h, l.files_offset - sizeof h) ||
        !all_zero(p + l.files_offset + l.files_bytes, l.descs_offset - l.files_offset - l.files_bytes) ||
        !all_zero(p + l.descs_offset + l.descs_bytes, l.bytes_offset - l.descs_offset - l.descs_bytes))
        return BAD;
    const uint8_t* region = p + l.bytes_offset;
    const uint32_t n_files = (uint32_t)h.n_files, n_frames = (uint32_t)h.n_frames;
    uint8_t fbytes[16];
    clx_frame_desc fd;
    const size_t flen = filler(h.nbytes, fbytes, &fd);
    if (flen == 0 || memcmp(region + h.nbytes, fbytes, flen) != 0 ||
        !all_zero(region + h.nbytes + flen, l.bytes_size - h.nbytes - flen))
        return BAD;
    std::vector<clx_frame_desc> descs(n_frames + 1);
    memcpy(descs.data(), p + l.descs_offset, l.descs_bytes);
    if (memcmp(&descs[n_frames], &fd, sizeof fd) != 0 || !corpus_frames_ok(region, h.nbytes, descs.data(), n_frames))
        return BAD;
    for (uint32_t f = 0; f < n_frames; f++)
        if (descs[f].out_offset != 0 || (descs[f].flags & ~(CLX_FRAME_VARIABLE_BLOCKING | CLX_FRAME_CRC16_VERIFIED)))
            return BAD;
    std::vector<uint32_t> file_frames(1, 0);
    std::vector<int32_t> tail;
    uint64_t base = 0;
    uint32_t frame = 0;
    for (uint32_t i = 0; i < n_files; i++) {
        const uint8_t* raw = p + l.files_offset + (uint64_t)i * sizeof(clx_image_file);
        clx_image_file r;
        memcpy(&r, raw, sizeof r);
        if (!all_zero(raw + INFO_PAD, 4) || r.byte_base != base || r.first_frame != frame ||
            r.n_frames > n_frames - frame || r.byte_count > h.nbytes - base || (r.flags & ~CLX_IMAGE_END_CONFIRMED))
            return BAD;
        if (r.n_frames == 0) {
            if (r.byte_count != 0 || r.flags != CLX_IMAGE_END_CONFIRMED || r.tail != CLX_OK) return BAD;
        } else {
            const clx_frame_desc* d = &descs[frame];
            const clx_frame_desc& last = d[r.n_frames - 1];
            // byte order keeps every frame at or after the first, which starts the file's bytes
            if (d[0].byte_offset != base || !file_frames_ok(d, r.n_frames) ||
                last.byte_offset + last.byte_len > base + r.byte_count)
                return BAD;
            const bool confirmed = last.flags & CLX_FRAME_CRC16_VERIFIED;
            if (r.flags != (confirmed ? CLX_IMAGE_END_CONFIRMED : 0u) ||
                (r.tail != CLX_OK && (confirmed || r.tail < CLX_ERR_IO_UNEXPECTED_EOF || r.tail > CLX_ERR_NO_BPS_IN_HEADER)))
                return BAD;
        }
        base += r.byte_count;
        frame += r.n_frames;
        file_frames.push_back(frame);
        tail.push_back(r.tail);
    }
    if (base != h.nbytes || frame != n_frames) return BAD;
    if (ix) {
        ix->bytes_offset = l.bytes_offset;
        ix->bytes_size = l.bytes_size;
        ix->nbytes = h.nbytes;
        ix->descs = std::move(descs);
        ix->file_frames = std::move(file_frames);
        ix->tail = std::move(tail);
    }
    return CLX_OK;
}

}  // namespace clx

extern "C" {

size_t clx_corpus_image_bytes(const size_t* file_nbytes, const clx_frame_desc* descs, size_t n_frames,
                              const uint32_t* file_frames, size_t n_files) {
    uint64_t nbytes;
    Layout l;
    if (!region_bytes(file_nbytes, descs, n_frames, file_frames, n_files, &nbytes) || !layout(n_files, n_frames, nbytes, &l))
        return 0;
    return (size_t)l.total;
}

int clx_corpus_image_write(clx_ctx* ctx, const uint8_t* const* file_bytes, const size_t* file_nbytes,
                           const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                           const clx_streaminfo* infos, void* image, size_t image_bytes) {
    uint64_t nbytes;
    Layout l;
    if (!ctx || !image || (n_files && (!file_bytes || !infos)) ||
        !region_bytes(file_nbytes, descs, n_frames, file_frames, n_files, &nbytes) || !layout(n_files, n_frames, nbytes, &l) ||
        image_bytes != l.total)
        return CLX_ERR_INVALID_ARGUMENT;
    for (size_t i = 0; i < n_files; i++) {
        const size_t n = file_frames[i + 1] - file_frames[i];
        if (n && !(clx::corpus_frames_ok(file_bytes[i], file_nbytes[i], descs + file_frames[i], n) &&
                   file_frames_ok(descs + file_frames[i], n)))
            return CLX_ERR_INVALID_ARGUMENT;
    }
    std::vector<int32_t> tail(n_files, CLX_OK);
    for (size_t i = 0; i < n_files; i++) {
        if (file_frames[i + 1] == file_frames[i]) continue;
        const clx_frame_desc& last = descs[file_frames[i + 1] - 1];
        if (!(last.flags & CLX_FRAME_CRC16_VERIFIED)) {
            const int rc = clx::tail_verdict(ctx, file_bytes[i], file_nbytes[i], last, &tail[i]);
            if (rc) return rc;
        }
    }
    uint8_t* p = static_cast<uint8_t*>(image);
    memset(p, 0, l.bytes_offset);  // header (its magic 0 until the end), records, descriptors and the gaps
    uint8_t* region = p + l.bytes_offset;
    uint64_t base = 0;
    for (size_t i = 0; i < n_files; i++) {
        clx_image_file r;
        memset(&r, 0, sizeof r);
        r.info = infos[i];
        memset(reinterpret_cast<uint8_t*>(&r) + INFO_PAD, 0, 4);
        r.byte_base = base;
        r.first_frame = file_frames[i];
        r.n_frames = file_frames[i + 1] - file_frames[i];
        r.flags = CLX_IMAGE_END_CONFIRMED;
        r.tail = tail[i];
        if (r.n_frames) {
            const uint64_t first = descs[file_frames[i]].byte_offset;
            r.byte_count = file_nbytes[i] - first;
            if (!(descs[file_frames[i + 1] - 1].flags & CLX_FRAME_CRC16_VERIFIED)) r.flags = 0;
            memcpy(region + base, file_bytes[i] + first, r.byte_count);
            for (size_t f = file_frames[i]; f < file_frames[i + 1]; f++) {
                clx_frame_desc d = descs[f];
                d.byte_offset = d.byte_offset - first + base;
                d.out_offset = 0;
                memcpy(p + l.descs_offset + f * sizeof d, &d, sizeof d);
            }
        }
        memcpy(p + l.files_offset + i * sizeof r, &r, sizeof r);
        base += r.byte_count;
    }
    uint8_t fbytes[16];
    clx_frame_desc fd;
    const size_t flen = filler(nbytes, fbytes, &fd);
    memcpy(p + l.descs_offset + n_frames * sizeof fd, &fd, sizeof fd);
    memcpy(region + nbytes, fbytes, flen);
    memset(region + nbytes + flen, 0, l.bytes_size - nbytes - flen);
    clx_image_header h;
    memset(&h, 0, sizeof h);
    h.version = CLX_IMAGE_VERSION;
    h.header_bytes = sizeof h;
    h.n_files = n_files;
    h.n_frames = n_frames;
    h.files_offset = l.files_offset;
    h.files_bytes = l.files_bytes;
    h.descs_offset = l.descs_offset;
    h.descs_bytes = l.descs_bytes;
    h.bytes_offset = l.bytes_offset;
    h.bytes_size = l.bytes_size;
    h.nbytes = nbytes;
    h.total_bytes = l.total;
    memcpy(p, &h, sizeof h);
    std::atomic_thread_fence(std::memory_order_release);  // everything above before the magic
    const uint64_t magic = CLX_IMAGE_MAGIC;
    memcpy(p, &magic, sizeof magic);
    return CLX_OK;
}

int clx_corpus_image_check(const void* image, size_t image_bytes) { return clx::read_image(image, image_bytes, nullptr); }

}  // extern "C"
