// clx_crops.cu — crop batches (include/claxon_b200.h, clx_batch_create_crops): [B, C, L] excerpts of a corpus in device
// or pinned host memory, planned on the device inside the batch's graph; and packed batches (clx_batch_create_packed),
// which lay variable-length excerpts along the columns of one [C, T] output.  A crop batch is a packed batch whose
// excerpts each own a row group: every kernel below is written once, templated on the layout (CropLayout or
// PackedLayout, clx_scan.cuh), which alone knows how a request reads, where an excerpt's output starts and whether it
// fits, what is zeroed around it and where unused slots go.
//
// The graph: the planner, then clx::launch_decode over every slot (with the device CRC-16), then the status pass.
//   1. excerpt_count_kernel: per excerpt, validate the request and binary-search the file's frame starts for the frames
//      that overlap [offset, offset + n) (plan_range in claxon_b200/__init__.py does the same on the host).
//   2. excerpt_scan_kernel: one CTA, the layout's start and fit of each excerpt, then exclusive scans of the slots (so
//      excerpts take consecutive slots in order and frames in stream order, the device order of load_crops()'s
//      windowed batch on a corpus of one shape), of the staging bytes and of the gather chunks.
//   2b. excerpt_gather_kernel, host corpora only: copies each excerpt's span of consecutive frames from mapped host
//      memory into its span of the batch's staging buffer.
//   3. excerpt_emit_kernel: per slot, the frame's descriptor (out_offset = its place in the planar scratch; over a host
//      corpus, byte_offset = its place in the staging buffer), its column on the excerpt's first row and its window.
//      Slots past the total go to the layout's trash: up to the next multiple of 32 they repeat the last planned
//      frame, after that they get the filler frame, so fillers share warps only with each other; no window has count 0.
//   4. excerpt_zero_kernel: zeroes exactly what no window of this call covers; the output is never cleared as a whole.
//   5. excerpt_status_kernel, after the decode: per excerpt the first failed slot, else the trailing-bytes verdict.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_scan.cuh"

namespace clx {

constexpr uint32_t CROP_THREADS = 256;

// The frames of a file, [f0, f1), that overlap its samples [lo, hi), lo < hi <= its length: the first of them in
// *first, their number returned (plan_range in claxon_b200/__init__.py does the same on the host).
__device__ __forceinline__ uint32_t overlapping_frames(const CropCorpus& cc, uint32_t f0, uint32_t f1, int64_t lo, int64_t hi,
                                                       uint32_t* first) {
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
    *first = i0;
    return a - i0;
}

// The last b < n with scan[b] <= x, scan ascending: the owner of slot (or chunk) x (owners without any own none).
__device__ __forceinline__ uint32_t owner_of(const uint32_t* scan, uint32_t n, uint32_t x) {
    uint32_t a = 0, e = n;
    while (e - a > 1) {
        const uint32_t m = (a + e) >> 1;
        if (scan[m] <= x) a = m;
        else e = m;
    }
    return a;
}

// Excerpts at or past the layout's used() are unused: status CLX_OK, length 0, no frames.
template <class Layout>
__global__ void __launch_bounds__(CROP_THREADS)
excerpt_count_kernel(CropCorpus cc, ExcerptBuffers eb) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b >= eb.n) return;
    const Layout at{eb};
    ExcerptPlan p{0, 0, 0, 0, 0};
    int64_t len = 0;
    int32_t st = CLX_OK;
    if (b < at.used()) {
        const clx_packed_request r = at.request(b);
        const int64_t n = request_ok(r, cc.n_files) ? excerpt_length(r, cc.file_len[r.file]) : -1;
        if (n < 0) {
            st = CLX_ERR_INVALID_ARGUMENT;
        } else {
            len = n;
            p = ExcerptPlan{r.offset, 0, 0, r.file, cc.file_ch[r.file]};
            if (len > 0)  // then the file has frames, and offset < its length
                p.count = overlapping_frames(cc, cc.file_frames[r.file], cc.file_frames[r.file + 1], r.offset,
                                             r.offset + len, &p.first);
        }
    }
    eb.plan[b] = p;
    eb.lengths[b] = len;
    eb.status[b] = st;
}

// Every load is a PCIe round trip of the order of a microsecond, so the grid keeps many in flight: a CTA copies
// GATHER_CHUNK bytes of one excerpt's span, each thread GATHER_VECS independent 16-byte loads before its stores.
constexpr uint32_t GATHER_THREADS = 256;
constexpr uint32_t GATHER_VECS = 4;
constexpr uint64_t GATHER_CHUNK = (uint64_t)GATHER_THREADS * GATHER_VECS * 16;

// One CTA, SCAN_THREADS excerpts at a time.  First the layout's start and fit of each valid excerpt (a packed batch's
// start_b is the scan of round_up_4(n_b), and an excerpt fits when start_b + n_b <= T; a crop always fits).  Then the
// slots of the excerpts that fit; one whose slots would pass n_slots does not fit either (never the case: n_slots bounds
// every call's frames; this keeps every later write in bounds whatever the requests).  Both rules leave the excerpts
// that fit a prefix of the valid ones.  Over a host corpus, each excerpt that fits and has frames takes span + 15
// staging bytes, its span starting at the first address of the same residue mod 16 as its source, and ceil(span /
// GATHER_CHUNK) gather chunks.
template <class Layout>
__global__ void __launch_bounds__(SCAN_THREADS)
excerpt_scan_kernel(CropCorpus cc, ExcerptBuffers eb) {
    __shared__ PackedSums s_warp[SCAN_THREADS / 32];
    __shared__ PackedSums s_cols, s_slots, s_final;
    __shared__ unsigned long long s_end;
    if (threadIdx.x == 0) s_cols = s_slots = s_final = PackedSums{}, s_end = 0;
    __syncthreads();
    const Layout at{eb};
    const uint32_t n = eb.n, used = at.used();
    for (uint32_t base = 0; base < n; base += SCAN_THREADS) {
        const uint32_t i = base + threadIdx.x;
        const bool valid = i < n && i < used && eb.status[i] == CLX_OK;
        const int64_t len = valid ? eb.lengths[i] : 0;
        const uint64_t start = at.start(i, len, s_warp, &s_cols);
        bool fit = valid && at.fits(start, len);
        const ExcerptPlan p = i < n ? eb.plan[i] : ExcerptPlan{};
        const uint32_t k = fit ? p.count : 0u;
        const uint32_t slot0 = cta_scan(PackedSums{0, 0, k, 0}, s_warp, &s_slots).slots;  // (every thread scans)
        fit = fit && slot0 + k <= eb.n_slots;
        uint64_t span = 0, s0 = 0;
        if (fit && p.count && cc.host_bytes) {
            s0 = cc.descs[p.first].byte_offset;
            const clx_frame_desc& last = cc.descs[p.first + p.count - 1];
            span = last.byte_offset + last.byte_len - s0;
        }
        const PackedSums mine{0, span ? span + 15 : 0, fit ? p.count : 0u,
                              span ? (uint32_t)((span + GATHER_CHUNK - 1) / GATHER_CHUNK) : 0u};
        const PackedSums sum = cta_scan(mine, s_warp, &s_final);
        if (i < n) {
            eb.scan[i] = sum.slots;
            eb.chunks[i] = sum.chunks;
            eb.stage[i] = sum.bytes + ((s0 - sum.bytes) & 15);
            if (valid && !fit) {
                eb.status[i] = CLX_ERR_INVALID_ARGUMENT;
                eb.lengths[i] = 0;
            }
            if (fit && len > 0) atomicMax(&s_end, (unsigned long long)at.end(start, len));
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        eb.scan[n] = s_final.slots;
        eb.chunks[n] = s_final.chunks;
        at.set_end(s_end);
    }
}

// Grid-stride over the chunks of every span: chunk k belongs to the excerpt whose chunk range holds it, CTA cx of the
// gx chunks of that span.  Source bytes [s0, s1) go to staging[x + delta], where x + delta and x agree mod 16: 16-byte
// vectors between a scalar head and tail (copied by cx 0).
__global__ void __launch_bounds__(GATHER_THREADS)
excerpt_gather_kernel(CropCorpus cc, ExcerptBuffers eb, uint8_t* __restrict__ staging) {
    const uint32_t total = eb.chunks[eb.n];
    for (uint32_t k = blockIdx.x; k < total; k += gridDim.x) {
        const uint32_t b = owner_of(eb.chunks, eb.n, k);
        const ExcerptPlan p = eb.plan[b];
        const uint64_t s0 = cc.descs[p.first].byte_offset;
        const clx_frame_desc& last = cc.descs[p.first + p.count - 1];
        const uint64_t s1 = last.byte_offset + last.byte_len, delta = eb.stage[b] - s0;
        const uint32_t cx = k - eb.chunks[b], gx = eb.chunks[b + 1] - eb.chunks[b];
        uint64_t a = (s0 + 15) & ~(uint64_t)15, e = s1 & ~(uint64_t)15;  // the vector part [a, e)
        if (e < a) a = e = s1;                                            // within one 16-byte block: all head
        if (cx == 0 && threadIdx.x < 32) {  // head [s0, a) on threads 0-15, tail [e, s1) on 16-31
            const uint64_t x = threadIdx.x < 16 ? s0 + threadIdx.x : e + (threadIdx.x - 16);
            if (x < (threadIdx.x < 16 ? a : s1)) staging[x + delta] = cc.host_bytes[x];
        }
        const uint4* src = reinterpret_cast<const uint4*>(cc.host_bytes + a);
        uint4* dst = reinterpret_cast<uint4*>(staging + (a + delta));
        const uint64_t nv = (e - a) >> 4;
        for (uint64_t v = (uint64_t)cx * GATHER_THREADS * GATHER_VECS + threadIdx.x; v < nv;
             v += (uint64_t)gx * GATHER_THREADS * GATHER_VECS) {
            uint4 r[GATHER_VECS];
#pragma unroll
            for (uint32_t j = 0; j < GATHER_VECS; j++)
                if (v + j * GATHER_THREADS < nv) r[j] = src[v + j * GATHER_THREADS];
#pragma unroll
            for (uint32_t j = 0; j < GATHER_VECS; j++)
                if (v + j * GATHER_THREADS < nv) dst[v + j * GATHER_THREADS] = r[j];
        }
    }
}

// Slot s: the frame's descriptor (out_offset = its place in the planar scratch; over a host corpus, byte_offset = its
// place in the staging buffer), its column on row 0 and its window.
template <class Layout>
__global__ void __launch_bounds__(CROP_THREADS)
excerpt_emit_kernel(CropCorpus cc, ExcerptBuffers eb, clx_frame_desc* __restrict__ descs, uint64_t* __restrict__ cols,
                    uint32_t* __restrict__ wins) {
    const uint32_t s = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (s >= eb.n_slots) return;
    const Layout at{eb};
    const uint32_t total = eb.scan[eb.n];
    clx_frame_desc d;
    uint64_t col;
    uint32_t win;
    // Unused slots in the last 32-slot group that holds planned frames repeat the last planned frame; the ones after it
    // get the filler frame.  Both go to the trash.  (The decode pass runs 32 frames per warp group: a filler next to
    // full-size frames takes the whole warp off its fast path, measured +1.1 ms per call at 176 400-sample crops.)
    const uint32_t slot = s < total ? s : s < ((total + 31) & ~31u) ? total - 1 : UINT32_MAX;
    if (slot == UINT32_MAX) {
        d = cc.descs[cc.n_frames];
        if (cc.staging) d.byte_offset = cc.staging;  // staged there at creation
    } else {
        const uint32_t b = owner_of(eb.scan, eb.n, slot);
        const ExcerptPlan p = eb.plan[b];
        const uint32_t f = p.first + (slot - eb.scan[b]);
        d = cc.descs[f];
        if (cc.staging)  // where the gather put the frame: its excerpt's span base plus its place in the span
            d.byte_offset = eb.stage[b] + (d.byte_offset - cc.descs[p.first].byte_offset);
        const int64_t s0 = cc.starts[f], hi = p.lo + eb.lengths[b];
        const int64_t first = max(p.lo - s0, (int64_t)0);
        const int64_t count = min(s0 + (int64_t)d.block_size, hi) - s0 - first;
        col = at.origin(b) + (uint64_t)(s0 + first - p.lo);
        win = (uint32_t)first | ((uint32_t)count << 16);
    }
    if (s >= total) {  // the whole frame (at most trash_width samples of it) on the trash
        col = at.trash();
        win = (uint32_t)(at.trash_width() < d.block_size ? at.trash_width() : d.block_size) << 16;
    }
    d.out_offset = (uint64_t)s * eb.slot_elems;
    descs[s] = d;
    cols[s] = col;
    wins[s] = win;
}

// One CTA row at a time (grid-stride over the (excerpt, row) pairs, then C rows after the excerpts), its threads over
// the layout's zero range of that row.
template <class Layout>
__global__ void __launch_bounds__(CROP_THREADS)
excerpt_zero_kernel(ExcerptBuffers eb, int32_t* __restrict__ out) {
    const Layout at{eb};
    const uint64_t rows = (uint64_t)(eb.n + 1) * eb.C;
    for (uint64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const uint32_t b = (uint32_t)(r / eb.C), c = (uint32_t)(r - (uint64_t)b * eb.C);
        uint64_t from, to;
        at.zero(b, c, &from, &to);
        int32_t* row = out + c * eb.L;
        for (uint64_t t = from + blockIdx.y * CROP_THREADS + threadIdx.x; t < to; t += (uint64_t)CROP_THREADS * gridDim.y)
            row[t] = 0;
    }
}

// Excerpt b's status after the decode: the planner's (an invalid request), else its first failed slot, else the
// trailing-bytes verdict; the error word keeps the smallest failure.
template <class Layout>
__global__ void __launch_bounds__(CROP_THREADS)
excerpt_status_kernel(CropCorpus cc, ExcerptBuffers eb, const clx_frame_result* __restrict__ results) {
    const uint32_t b = blockIdx.x * CROP_THREADS + threadIdx.x;
    if (b == 0) Layout{eb}.keep_end();
    if (b >= eb.n) return;
    int32_t st = eb.status[b];
    unsigned long long kind = 0;
    if (st == CLX_OK) {
        const uint32_t s0 = eb.scan[b], s1 = eb.scan[b + 1];
        for (uint32_t s = s0; s < s1 && st == CLX_OK; s++) st = results[s].status;
        kind = 1;
        if (st == CLX_OK && s1 > s0) {  // an unconfirmed last frame inside the excerpt: what follows it
            const ExcerptPlan p = eb.plan[b];
            const uint32_t last = cc.file_frames[p.file + 1] - 1;
            if (cc.file_tail[p.file] != CLX_OK && p.lo + eb.lengths[b] > cc.starts[last]) {
                st = cc.file_tail[p.file];
                kind = 2;
            }
        }
        eb.status[b] = st;
    }
    if (st != CLX_OK) atomicMin(eb.error, (kind << 62) | ((unsigned long long)b << 32) | (uint32_t)st);
}

template <class Layout>
cudaError_t launch_excerpts(const CropCorpus& cc, const ExcerptBuffers& eb, const DecodeBuffers& db, const Plan& plan,
                            bool crc, cudaStream_t stream, uint64_t* launches) {
    cudaError_t e = cudaMemsetAsync(eb.error, 0xff, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const uint32_t ctas = (eb.n + CROP_THREADS - 1) / CROP_THREADS;
    excerpt_count_kernel<Layout><<<ctas, CROP_THREADS, 0, stream>>>(cc, eb);
    excerpt_scan_kernel<Layout><<<1, SCAN_THREADS, 0, stream>>>(cc, eb);
    if (cc.host_bytes) {
        // every span's chunks together: ceil(span / GATHER_CHUNK) per excerpt, the spans within the staging size
        const uint32_t chunks = (uint32_t)std::min<uint64_t>(cc.staging / GATHER_CHUNK + eb.n, 1u << 20);
        excerpt_gather_kernel<<<chunks, GATHER_THREADS, 0, stream>>>(cc, eb, const_cast<uint8_t*>(db.bytes));
        (*launches)++;
    }
    excerpt_emit_kernel<Layout><<<(eb.n_slots + CROP_THREADS - 1) / CROP_THREADS, CROP_THREADS, 0, stream>>>(
        cc, eb, const_cast<clx_frame_desc*>(db.descs), const_cast<uint64_t*>(db.cols), const_cast<uint32_t*>(db.wins));
    const uint64_t rows = (uint64_t)(eb.n + 1) * eb.C;
    const dim3 zgrid((uint32_t)std::min<uint64_t>(rows, 32768),
                     (uint32_t)std::min<uint64_t>((Layout{eb}.width() + 8191) / 8192, 16));
    excerpt_zero_kernel<Layout><<<zgrid, CROP_THREADS, 0, stream>>>(eb, static_cast<int32_t*>(db.conv));
    *launches += 4;
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    e = launch_decode(db, plan, crc, stream, launches);
    if (e != cudaSuccess) return e;
    excerpt_status_kernel<Layout><<<ctas, CROP_THREADS, 0, stream>>>(cc, eb, db.results);
    (*launches)++;
    return cudaGetLastError();
}
template cudaError_t launch_excerpts<CropLayout>(const CropCorpus&, const ExcerptBuffers&, const DecodeBuffers&,
                                                 const Plan&, bool, cudaStream_t, uint64_t*);
template cudaError_t launch_excerpts<PackedLayout>(const CropCorpus&, const ExcerptBuffers&, const DecodeBuffers&,
                                                   const Plan&, bool, cudaStream_t, uint64_t*);

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

size_t clx_packed_frames_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                               size_t max_excerpts, size_t max_samples) {
    if (max_excerpts == 0 || max_samples == 0 || !file_frames || (!descs && n_frames) || file_frames[n_files] != n_frames)
        return 0;
    for (size_t i = 0; i < n_files; i++)
        if (file_frames[i + 1] < file_frames[i]) return 0;
    uint32_t m = 0;   // smallest block size of a frame that is not the last of its file (0: none)
    size_t most = 0;  // frames of the largest file
    for (size_t i = 0; i < n_files; i++) {
        most = std::max<size_t>(most, file_frames[i + 1] - file_frames[i]);
        for (size_t f = file_frames[i]; f + 1 < file_frames[i + 1]; f++)
            if (m == 0 || descs[f].block_size < m) m = descs[f].block_size;
    }
    // Excerpts that fit hold at most T samples in all, so at most k = min(B, T) of them have frames.  One of n samples
    // overlaps at most (n - 2) / m + 2 frames (the first and last give one sample or more, the ones between whole non-last
    // blocks; 1 <= 2 - 1 / m for n = 1), so all of them together floor((T - 2k) / m) + 2k, since the sum grows with k.
    const size_t k = std::min(max_excerpts, max_samples);
    if (m == 0) return k;
    const int64_t d = (int64_t)max_samples - 2 * (int64_t)k;  // (>= -T: no overflow)
    const int64_t q = d >= 0 ? d / m : -((-d + m - 1) / (int64_t)m);
    const size_t s = (size_t)(q + 2 * (int64_t)k);
    return std::max<size_t>(1, most && k <= SIZE_MAX / most ? std::min(s, k * most) : s);
}

size_t clx_packed_bytes_bound(const clx_frame_desc* descs, size_t n_frames, const uint32_t* file_frames, size_t n_files,
                              size_t max_excerpts, size_t max_samples) {
    const size_t S = clx_packed_frames_bound(descs, n_frames, file_frames, n_files, max_excerpts, max_samples);
    if (S == 0) return 0;
    // An excerpt's span, frames f .. g of one file: the advances from f to g plus byte_len(g), at most its frame count
    // times the largest per-frame advance (gaps between frames included), so every span together at most S times it.
    uint64_t adv = 0;
    for (size_t i = 0; i < n_files; i++)
        for (size_t f = file_frames[i]; f < file_frames[i + 1]; f++) {
            adv = std::max<uint64_t>(adv, descs[f].byte_len);
            if (f + 1 < file_frames[i + 1] && descs[f + 1].byte_offset > descs[f].byte_offset)
                adv = std::max<uint64_t>(adv, descs[f + 1].byte_offset - descs[f].byte_offset);
        }
    if (max_excerpts > SIZE_MAX / 32 || (adv && S > (SIZE_MAX - 16 * max_excerpts) / adv)) return SIZE_MAX;
    return S * adv + 16 * max_excerpts;
}

}  // extern "C"
