// clx_decode.cu — sm_90a frame-decode kernels of claxon_b200.
//
// What runs here is everything claxon does between the frame-header parse and the
// CRC-16 footer check of FrameReader::read_next_or_eof (reference src/frame.rs:701-742):
//   subframe::decode            src/subframe.rs:184-228   (header, wasted bits)
//   decode_constant / verbatim  src/subframe.rs:382-415
//   decode_fixed / decode_lpc   src/subframe.rs:492-516, :651-721 (warm-up, LPC parameters)
//   decode_residual, Rice/Rice2 src/subframe.rs:236-380
//   predict_fixed / predict_lpc src/subframe.rs:417-474, :524-614
//   decode_{left,right,mid}_side src/frame.rs:319-389
//
// Mapping (DESIGN.md §3): ONE LANE PER FRAME.  A FLAC frame is one continuous bitstream
// whose subframe and partition boundaries are only known after the preceding codes have
// been parsed, and the LPC synthesis is a strictly serial recurrence (the floor in
// `>> qlp_shift` makes it non-associative), so the parallel axis is the batch of
// independent frames: 32 frames advance per warp instruction, each lane owning the bit
// cursor, Rice state, predictor coefficients and the last `order` samples of its frame
// in registers.  Lanes run in lockstep on the *sample index*: every step each lane
// produces exactly one sample, so the decoded samples of a warp form a 32(frames) x
// 32(steps) tile that is staged through shared memory and written to HBM as coalesced
// 16-byte vectors (planar `Block` layout, src/frame.rs:477-481).  Inter-channel
// decorrelation happens in that write-out stage.
//
// All sample arithmetic is integer and bit-exact with the reference: i64 accumulate,
// arithmetic shift, truncating cast for LPC; wrapping i32 for fixed predictors, wasted
// bits and stereo decorrelation.  There is no floating point and no tensor-core work.
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

#include "claxon_b200.h"
#include "clx_internal.h"
#include "clx_lanes.h"

namespace clx {

constexpr int WARPS_PER_CTA = 4;
constexpr int TILE_WORDS = 32 * 32;  // one 32x32 i32 tile per warp

enum Mode : int { M_HEADER = 0, M_VERB = 1, M_RICE = 2, M_CONST = 3, M_DONE = 4 };

// ---------------------------------------------------------------------------------
// Bit cursor.  Semantics = claxon's Bitstream (src/input.rs:415-643): MSB-first bit fields.
//
// Frame bytes are staged from HBM into shared memory by the TMA engine: every lane owns a
// 128-byte ring (two 64-byte halves) in shared memory and a pair of mbarriers; when its cursor
// enters a new 64-byte chunk it waits for that chunk's mbarrier and immediately issues a
// `cp.async.bulk` (16-byte-aligned global source, SASS UBLKCP) for the following chunk, so a
// chunk is requested ~85 samples (several thousand cycles) before its first word is read and
// HBM latency never sits on the decode's critical path.  The cursor itself keeps three
// big-endian words of look-ahead in registers plus one raw word in flight from shared memory.
// Running past the frame's available bytes is detected by position (see `overrun`) and reported
// as UnexpectedEof; chunk requests are clamped to the buffer, never faulting.
// ---------------------------------------------------------------------------------
constexpr uint32_t RING_LANE_BYTES = 144;  // 2 x 64-byte halves + 16 bytes of bank skew (36 words: 4-way max)
constexpr uint32_t CHUNK_BYTES = 64;

struct BitCur {
    const uint8_t* gbase;  // 16-byte aligned global address at or before the frame's first byte
    uint32_t ring;         // shared-space address of this lane's ring
    uint32_t bars;         // shared-space address of this lane's two mbarriers
    uint32_t chunk_lim;    // highest chunk index that lies inside the byte buffer
    uint32_t widx;         // word index (from gbase) of the next word to load from the ring
    uint32_t cw0, cw1, cw2, raw;
    uint32_t off;          // 0..31: bits of cw0 already consumed
};

__device__ __forceinline__ void tma_request_chunk(const BitCur& b, uint32_t c) {
    const uint32_t bar = b.bars + (c & 1) * 8;
    const uint32_t dst = b.ring + (c & 1) * CHUNK_BYTES;
    const uint8_t* src = b.gbase + (size_t)min(c, b.chunk_lim) * CHUNK_BYTES;
    // order this thread's earlier generic-proxy reads of the half before the async-proxy write
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(CHUNK_BYTES) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
        "l"(src), "r"(CHUNK_BYTES), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void tma_wait_chunk(const BitCur& b, uint32_t c) {
    const uint32_t bar = b.bars + (c & 1) * 8;
    const uint32_t parity = (c >> 1) & 1;
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ uint32_t ring_load(const BitCur& b, uint32_t w) {
    uint32_t x;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(b.ring + ((w & 31u) << 2)) : "memory");
    return x;
}
__device__ __forceinline__ uint32_t bc_fetch(BitCur& b) {
    if ((b.widx & 15u) == 0) {  // first word of a chunk: it must have landed; prefetch the next one
        const uint32_t c = b.widx >> 4;
        tma_wait_chunk(b, c);
        tma_request_chunk(b, c + 1);
    }
    uint32_t x = b.raw;
    b.raw = ring_load(b, b.widx);
    b.widx++;
    return __byte_perm(x, 0, 0x0123);
}
// `smem_ring` / `smem_bars`: generic pointers to this lane's ring and mbarrier pair.
__device__ __forceinline__ void bc_init(BitCur& b, const uint8_t* bytes, uint64_t byte_off, uint64_t buf_bytes,
                                        uint32_t start_bit, void* smem_ring, void* smem_bars) {
    const uint64_t aligned = byte_off & ~15ull;
    b.gbase = bytes + aligned;
    b.ring = (uint32_t)__cvta_generic_to_shared(smem_ring);
    b.bars = (uint32_t)__cvta_generic_to_shared(smem_bars);
    const uint64_t chunks = (buf_bytes - aligned) / CHUNK_BYTES;  // buffer is padded: >= 2
    b.chunk_lim = (uint32_t)min(chunks - 1, (uint64_t)0x3fffffu);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b.bars) : "memory");
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b.bars + 8) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint32_t bit = (uint32_t)(byte_off & 15) * 8 + start_bit;
    const uint32_t s = bit >> 5;
    b.off = bit & 31;
    uint32_t c = s >> 4;
    tma_request_chunk(b, c);
    tma_wait_chunk(b, c);
    tma_request_chunk(b, c + 1);
    uint32_t w[4];
#pragma unroll
    for (uint32_t i = 0; i < 4; i++) {
        if (i > 0 && ((s + i) & 15u) == 0) {
            tma_wait_chunk(b, (s + i) >> 4);
            tma_request_chunk(b, ((s + i) >> 4) + 1);
        }
        w[i] = ring_load(b, s + i);
    }
    b.cw0 = __byte_perm(w[0], 0, 0x0123);
    b.cw1 = __byte_perm(w[1], 0, 0x0123);
    b.cw2 = __byte_perm(w[2], 0, 0x0123);
    b.raw = w[3];
    b.widx = s + 4;
}
// Bits consumed so far, relative to gbase.
__device__ __forceinline__ uint32_t bc_pos(const BitCur& b) { return (b.widx - 4) * 32 + b.off; }
__device__ __forceinline__ uint32_t bc_peek(const BitCur& b) { return __funnelshift_l(b.cw1, b.cw0, b.off); }
__device__ __forceinline__ void bc_skip(BitCur& b, uint32_t n) {  // n <= 32
    b.off += n;
    if (b.off >= 32) {
        b.off -= 32;
        b.cw0 = b.cw1;
        b.cw1 = b.cw2;
        b.cw2 = bc_fetch(b);
    }
}
__device__ __forceinline__ uint32_t bc_read(BitCur& b, uint32_t n) {  // n <= 32
    uint32_t hi = bc_peek(b);
    uint32_t v = __funnelshift_l(hi, 0, n & 31);  // top n bits (n<32)
    if (n == 32) v = hi;
    bc_skip(b, n);
    return v;
}
// Unary run of any length (src/input.rs:475-511); stops counting once past `limit_bits`.
__device__ __forceinline__ uint32_t bc_unary_slow(BitCur& b, uint32_t limit_bits) {
    uint32_t q = 0;
    for (;;) {
        uint32_t hi = bc_peek(b);
        if (hi != 0) {
            uint32_t z = __clz(hi);
            q += z;
            bc_skip(b, z + 1);
            return q;
        }
        q += 32;
        bc_skip(b, 32);
        if (bc_pos(b) > limit_bits) return q;  // ran off the frame: caller reports UnexpectedEof
    }
}

// ---------------------------------------------------------------------------------
// Shared-memory staging tile, one per warp: row = lane (frame), 32 columns = 32 consecutive
// steps.  16-byte groups are XOR-swizzled by (row & 7) so that both the per-lane 16-byte
// stores (8 lanes -> 8 rows per phase) and the row-wise 16-byte loads are conflict free.
// ---------------------------------------------------------------------------------
struct RowInfo {      // per lane/frame, constant for the kernel
    int32_t* out;     // frame's first output element
    uint32_t total;   // n_channels * block_size
    uint32_t bs_mode; // block_size | channel_assignment << 16 | vec_ok << 24
};

// Inter-channel decorrelation of one (ch0, ch1) pair; wrapping i32 (src/frame.rs:319-389).
__device__ __forceinline__ void decorrelate(uint32_t ca, int32_t a, int32_t b, int32_t& o0, int32_t& o1) {
    if (ca == 8) {  // left/side: right = left - side
        o0 = a;
        o1 = (int32_t)((uint32_t)a - (uint32_t)b);
    } else if (ca == 9) {  // side/right: left = side + right
        o0 = (int32_t)((uint32_t)a + (uint32_t)b);
        o1 = b;
    } else {  // mid/side; (mid*2|side&1) +- side is even, so the reference's `/ 2` == `>> 1`
        uint32_t m = ((uint32_t)a << 1) | ((uint32_t)b & 1u);
        o0 = ((int32_t)(m + (uint32_t)b)) >> 1;
        o1 = ((int32_t)(m - (uint32_t)b)) >> 1;
    }
}

// Writes the warp's tile (steps [g0, g0+32)) to global memory.
__device__ __noinline__ void flush_tile(const int32_t* tile, const RowInfo* rows, uint32_t g0, uint32_t lane) {
    __syncwarp();
    // ---- vector pass: 4 rows per iteration, 8 lanes x 16 bytes per row ----
    uint32_t slow_rows = 0;
#pragma unroll 2
    for (uint32_t pass = 0; pass < 8; pass++) {
        uint32_t r = pass * 4 + (lane >> 3), grp = lane & 7;
        RowInfo ri = rows[r];
        uint32_t bs = ri.bs_mode & 0xffffu, ca = (ri.bs_mode >> 16) & 0xffu, vec_ok = ri.bs_mode >> 24;
        bool live = g0 < ri.total;
        bool fast = live && vec_ok && (g0 + 32 <= ri.total);
        uint32_t g = g0 + grp * 4;
        if (fast) {
            int4 v = *reinterpret_cast<const int4*>(tile + r * 32 + ((grp ^ (r & 7)) << 2));
            if (ca >= 8 && g >= bs) {  // second channel of a decorrelated pair: vec_ok => bs % 32 == 0
                int4* p0 = reinterpret_cast<int4*>(ri.out + (g - bs));
                int4 a = __ldcg(p0);
                int4 o0, o1;
                decorrelate(ca, a.x, v.x, o0.x, o1.x);
                decorrelate(ca, a.y, v.y, o0.y, o1.y);
                decorrelate(ca, a.z, v.z, o0.z, o1.z);
                decorrelate(ca, a.w, v.w, o0.w, o1.w);
                if (ca != 8) *p0 = o0;
                *reinterpret_cast<int4*>(ri.out + g) = o1;
            } else {
                *reinterpret_cast<int4*>(ri.out + g) = v;
            }
        }
        uint32_t slow = __ballot_sync(0xffffffffu, live && !fast);
        // lanes 0,8,16,24 carry the verdict of rows pass*4 .. pass*4+3
        slow_rows |= (((slow >> 0) & 1u) | (((slow >> 8) & 1u) << 1) | (((slow >> 16) & 1u) << 2) |
                      (((slow >> 24) & 1u) << 3))
                     << (pass * 4);
    }
    // ---- scalar passes for rows that are ragged, unaligned or straddle channels ----
    if (slow_rows) {
        for (int phase = 0; phase < 2; phase++) {
            uint32_t todo = slow_rows;
            while (todo) {
                uint32_t r = __ffs(todo) - 1;
                todo &= todo - 1;
                RowInfo ri = rows[r];
                uint32_t bs = ri.bs_mode & 0xffffu, ca = (ri.bs_mode >> 16) & 0xffu;
                uint32_t g = g0 + lane;
                if (g < ri.total) {
                    int32_t v = tile[tile_word(r, lane)];
                    bool second = ca >= 8 && g >= bs;
                    if (phase == 0 && !second) ri.out[g] = v;
                    if (phase == 1 && second) {
                        int32_t a = __ldcg(ri.out + (g - bs)), o0, o1;
                        decorrelate(ca, a, v, o0, o1);
                        ri.out[g - bs] = o0;
                        ri.out[g] = o1;
                    }
                }
            }
            __syncwarp();  // phase 1 reads first-channel samples that phase 0 may just have written
        }
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------------
// Per-lane decoder state
// ---------------------------------------------------------------------------------
template <int KORD>
struct Lane {
    BitCur bc;
    uint32_t limit_bits;   // bits available to the frame, relative to bc.base
    uint32_t frame_bit0;   // bit position of the frame's first byte, relative to bc.base
    uint32_t bs, nch, ca, bps, total;
    uint32_t ch;           // current subframe
    uint32_t t;            // samples produced in the current subframe
    int mode;
    uint32_t order, wasted, sfbps;
    bool pred;             // fixed or LPC subframe
    bool is_lpc;
    bool params_done;
    uint32_t shift;        // qlp shift (0 for fixed)
    uint32_t k, rem, parts_left, per, pbits;  // Rice state
    int32_t cval;
    int32_t status;
    int32_t h[KORD];       // h[KORD-1] = most recent sample
    int32_t c[KORD];       // c[j] multiplies h[j]; zero for taps older than `order`
};

template <int KORD>
__device__ __forceinline__ bool overrun(const Lane<KORD>& L) { return bc_pos(L.bc) > L.limit_bits; }

// Enter the error state: remaining samples of the frame are written as zero so that the
// output region is fully overwritten (never stale, cf. claxon changelog 0.4.1).
// An error found after the cursor ran past the frame's bytes is an UnexpectedEof that
// happened first in stream order (src/input.rs:139-142).
template <int KORD>
__device__ __forceinline__ void fail_at(Lane<KORD>& L, int code, uint32_t field_end) {
    // `field_end` = position just past the field whose value is being rejected: claxon would
    // have hit UnexpectedEof first iff that field does not fit in the frame's bytes.
    L.status = field_end > L.limit_bits ? (int)CLX_ERR_IO_UNEXPECTED_EOF : code;
    L.mode = M_CONST;
    L.cval = 0;
    L.wasted = 0;
    L.pred = false;
    L.ch = L.nch;  // no more subframes
    L.t = 0;
}
template <int KORD>
__device__ __forceinline__ void fail(Lane<KORD>& L, int code) { fail_at(L, code, bc_pos(L.bc)); }

// read_subframe_header + dispatch preamble (src/subframe.rs:29-91, :184-211, :382-394,
// :499-504, :662-667).
template <int KORD>
__device__ __forceinline__ void parse_subframe_header(Lane<KORD>& L, int* need_hi) {
    BitCur& b = L.bc;
    uint32_t bps = L.bps;
    if (L.ca == 9) bps += (L.ch == 0);                 // side/right: side first (src/frame.rs:725)
    else if (L.ca == 8 || L.ca == 10) bps += (L.ch == 1);  // src/frame.rs:717, :736
    const uint32_t p0 = bc_pos(b);
    uint32_t head = bc_read(b, 8);  // pad bit, 6-bit type, wasted-bits flag
    if (head & 0x80u) return fail_at(L, CLX_ERR_SUBFRAME_HEADER_INVALID, p0 + 1);
    uint32_t code = (head >> 1) & 0x3fu;
    L.pred = false;
    L.is_lpc = false;
    L.order = 0;
    int type;  // 0 const 1 verbatim 2 fixed 3 lpc
    if (code == 0) type = 0;
    else if (code == 1) type = 1;
    else if ((code & 0x3eu) == 0x02u || (code & 0x3cu) == 0x04u || (code & 0x30u) == 0x10u)
        return fail_at(L, CLX_ERR_SUBFRAME_HEADER_RESERVED, p0 + 7);
    else if ((code & 0x38u) == 0x08u) {
        L.order = code & 7u;
        if (L.order > 4) return fail_at(L, CLX_ERR_SUBFRAME_HEADER_RESERVED, p0 + 7);
        type = 2;
    } else {
        L.order = (code & 0x1fu) + 1;
        type = 3;
    }
    uint32_t wasted = 0;
    if (head & 1u) {
        uint32_t hi = bc_peek(b);
        uint32_t q;
        if (hi != 0) { q = __clz(hi); bc_skip(b, q + 1); }
        else q = bc_unary_slow(b, L.limit_bits);
        wasted = 1 + q;
    }
    if (overrun(L)) return fail(L, CLX_ERR_IO_UNEXPECTED_EOF);
    if (wasted > 31) return fail(L, CLX_ERR_WASTED_BITS_GT_31);
    if (wasted >= bps) return fail(L, CLX_ERR_NO_NON_WASTED_BITS);
    L.wasted = wasted;
    L.sfbps = bps - wasted;
    L.t = 0;
    L.params_done = false;
#pragma unroll
    for (int j = 0; j < KORD; j++) L.c[j] = 0;
    if (type == 0) {
        L.cval = hd_sext(bc_read(b, L.sfbps), L.sfbps);
        L.mode = M_CONST;
        if (overrun(L)) return fail(L, CLX_ERR_IO_UNEXPECTED_EOF);
    } else if (type == 1) {
        L.mode = M_VERB;
    } else {
        if (L.bs < L.order)
            return fail(L, type == 2 ? CLX_ERR_FIXED_ORDER_GT_BLOCK : CLX_ERR_LPC_ORDER_GT_BLOCK);
        if (L.order > (uint32_t)KORD) {  // this kernel instance keeps only KORD taps in registers
            *need_hi = 1;
            L.status = CLX_INTERNAL_NEED_HIGH_ORDER;
            L.mode = M_CONST; L.cval = 0; L.wasted = 0; L.ch = L.nch; L.t = 0;
            return;
        }
        L.pred = true;
        L.is_lpc = type == 3;
        L.mode = M_VERB;  // warm-up samples are verbatim (src/subframe.rs:504, :667)
    }
}

// Next Rice partition header (src/subframe.rs:314-319, :362-367).
template <int KORD>
__device__ __forceinline__ void next_partition(Lane<KORD>& L, uint32_t len) {
    uint32_t k = bc_read(L.bc, L.pbits);
    if (k == (1u << L.pbits) - 1u) return fail(L, CLX_ERR_UNENCODED_BINARY);
    L.k = k;
    L.rem = len;
    L.parts_left--;
}

// LPC parameters (src/subframe.rs:669-701) / fixed coefficient rows (:427-431), then the
// residual header (:241-277) and the first partition's parameter.
template <int KORD>
__device__ __forceinline__ void parse_params(Lane<KORD>& L) {
    BitCur& b = L.bc;
    L.params_done = true;
    if (L.is_lpc) {
        const uint32_t p0 = bc_pos(b);
        uint32_t pq = bc_read(b, 9);  // 4-bit precision-1, 5-bit signed shift
        uint32_t prec_m1 = pq >> 5;
        if (prec_m1 == 15) return fail_at(L, CLX_ERR_QLP_PRECISION_INVALID, p0 + 4);
        uint32_t precision = prec_m1 + 1;
        int32_t shift = hd_sext(pq & 31u, 5);
        if (shift < 0) return fail(L, CLX_ERR_NEGATIVE_QLP_SHIFT);
        L.shift = (uint32_t)shift;
        // First coefficient in the stream multiplies the most recent sample (:696-701).
#pragma unroll
        for (int j = KORD - 1; j >= 0; j--) {
            if ((uint32_t)(KORD - 1 - j) < L.order)
                L.c[j] = hd_sext(bc_read(b, precision), precision);
        }
    } else {
        L.shift = 0;
        // Rows of Pascal's triangle with alternating sign; c[KORD-1] multiplies s[i-1].
        const int32_t r1 = L.order == 1 ? 1 : L.order == 2 ? 2 : L.order == 3 ? 3 : L.order == 4 ? 4 : 0;
        const int32_t r2 = L.order == 2 ? -1 : L.order == 3 ? -3 : L.order == 4 ? -6 : 0;
        const int32_t r3 = L.order == 3 ? 1 : L.order == 4 ? 4 : 0;
        const int32_t r4 = L.order == 4 ? -1 : 0;
        L.c[KORD - 1] = r1;
        L.c[KORD - 2] = r2;
        L.c[KORD - 3] = r3;
        L.c[KORD - 4] = r4;
    }
    const uint32_t pr = bc_pos(b);
    uint32_t rh = bc_read(b, 6);  // 2-bit coding method, 4-bit partition order
    uint32_t method = rh >> 4, po = rh & 15u;
    if (method > 1) return fail_at(L, CLX_ERR_RESIDUAL_RESERVED, pr + 2);
    if (overrun(L)) return fail(L, CLX_ERR_IO_UNEXPECTED_EOF);
    uint32_t n_part = 1u << po;
    if ((L.bs & ((n_part - 1u) & 0xffffu)) != 0) return fail(L, CLX_ERR_PARTITION_ORDER_INVALID);
    L.per = L.bs >> po;
    if (L.order > L.per) return fail(L, CLX_ERR_RESIDUAL_INVALID);
    L.pbits = method == 0 ? 4u : 5u;
    L.parts_left = n_part;
    L.mode = M_RICE;
    next_partition(L, L.per - L.order);
    // An empty first partition still has its parameter read (src/subframe.rs:283-288).
    if (L.mode == M_RICE && L.rem == 0 && L.parts_left > 0) next_partition(L, L.per);
    if (L.mode == M_RICE && overrun(L)) return fail(L, CLX_ERR_IO_UNEXPECTED_EOF);
}

// One Rice/Rice2 code (src/subframe.rs:336-347, :369-377): q zeros, a one, k remainder bits;
// value (q << k) | r in wrapping u32, then the zig-zag map of rice_to_signed (:157-170).
template <int KORD>
__device__ __forceinline__ int32_t rice_decode(Lane<KORD>& L) {
    BitCur& b = L.bc;
    uint32_t hi = bc_peek(b);
    uint32_t q = __clz(hi);
    uint32_t n = q + 1 + L.k;
    uint32_t r;
    if (n <= 32) {
        uint32_t tt = (hi << q) << 1;
        r = __funnelshift_l(tt, 0, L.k);
        bc_skip(b, n);
    } else {
        q = bc_unary_slow(b, L.limit_bits);
        r = L.k ? bc_read(b, L.k) : 0u;
    }
    uint32_t u = (q << L.k) | r;
    return (int32_t)((u >> 1) ^ (0u - (u & 1u)));
}

// Prediction with TAPS taps out of the KORD kept: i64 accumulate, arithmetic shift,
// truncation to i32 (src/subframe.rs:576-581, :607-612).  Fixed predictors use the same
// path with shift 0: the i64 sum truncated to 32 bits equals the reference's wrapping
// i32 arithmetic (:461-470).
template <int KORD, int TAPS>
__device__ __forceinline__ int32_t predict(const int32_t (&v)[KORD + 4], int first, const int32_t (&c)[KORD],
                                           uint32_t shift) {
    long long acc = 0;
#pragma unroll
    for (int j = KORD - TAPS; j < KORD; j++) acc += (long long)c[j] * (long long)v[j + first];
    return (int32_t)(acc >> shift);
}

// ---------------------------------------------------------------------------------
// The kernel
// ---------------------------------------------------------------------------------
template <int KORD>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32)
decode_frames_kernel(const uint8_t* __restrict__ bytes, uint64_t buf_bytes,
                     const clx_frame_desc* __restrict__ descs, uint32_t n_frames,
                     int32_t* __restrict__ out, clx_frame_result* __restrict__ results,
                     int* __restrict__ need_hi, const int* __restrict__ gate, int select_status) {
    __shared__ __align__(16) int32_t s_tile[WARPS_PER_CTA][TILE_WORDS];
    __shared__ __align__(16) RowInfo s_rows[WARPS_PER_CTA][32];
    __shared__ __align__(16) uint8_t s_ring[WARPS_PER_CTA][32 * RING_LANE_BYTES];
    __shared__ __align__(8) uint64_t s_bars[WARPS_PER_CTA][32][2];

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t fidx = blockIdx.x * (WARPS_PER_CTA * 32) + threadIdx.x;
    int32_t* tile = s_tile[warp];
    RowInfo* rows = s_rows[warp];

    // select_status != 0: decode only the frames an earlier kernel marked with that status;
    // `gate` (if given) is that kernel's "anything marked?" word, so the common case exits at once.
    if (gate != nullptr && *gate == 0) return;

    Lane<KORD> L;
    L.status = CLX_OK;
    L.mode = M_DONE;
    L.total = 0;
    L.bs = 0; L.nch = 0; L.ca = 0; L.bps = 0; L.ch = 0; L.t = 0;
    L.order = 0; L.wasted = 0; L.sfbps = 0; L.pred = false; L.is_lpc = false; L.params_done = false;
    L.shift = 0; L.k = 0; L.rem = 0; L.parts_left = 0; L.per = 0; L.pbits = 4; L.cval = 0;
    L.limit_bits = 0; L.frame_bit0 = 0;
#pragma unroll
    for (int j = 0; j < KORD; j++) { L.h[j] = 0; L.c[j] = 0; }

    bool have = fidx < n_frames;
    if (have && select_status != 0) have = results[fidx].status == select_status;
    RowInfo ri;
    ri.out = out;
    ri.total = 0;
    ri.bs_mode = 0;
    uint32_t byte_len = 0;
    if (have) {
        clx_frame_desc d = descs[fidx];
        L.bs = d.block_size;
        L.nch = d.n_channels;
        L.ca = d.channel_assignment;
        L.bps = d.bits_per_sample;
        L.total = L.bs * L.nch;
        byte_len = d.byte_len;
        bc_init(L.bc, bytes, d.byte_offset, buf_bytes, (uint32_t)d.header_len * 8,
                s_ring[warp] + lane * RING_LANE_BYTES, &s_bars[warp][lane][0]);
        L.frame_bit0 = (uint32_t)(d.byte_offset & 15) * 8;
        L.limit_bits = L.frame_bit0 + byte_len * 8;
        L.mode = M_HEADER;
        ri.out = out + d.out_offset;
        ri.total = L.total;
        uint32_t vec_ok = ((d.out_offset & 3) == 0) && ((L.bs & 31) == 0);
        ri.bs_mode = L.bs | (L.ca << 16) | (vec_ok << 24);
        if (L.bps == 0) {  // src/frame.rs:687-692
            L.status = CLX_ERR_NO_BPS_IN_HEADER;
            L.mode = M_CONST; L.cval = 0; L.ch = L.nch;
        }
    }
    if (!have)  // idle lanes follow the same cursor protocol over the start of the buffer (never decoded)
        bc_init(L.bc, bytes, 0, buf_bytes, 0, s_ring[warp] + lane * RING_LANE_BYTES, &s_bars[warp][lane][0]);
    rows[lane] = ri;
    __syncwarp();

    const uint32_t steps = __reduce_max_sync(0xffffffffu, L.total);

    // Frame end (runs once per lane, as soon as its last sample has been produced — later the
    // lane keeps executing the warp's instruction stream with its cursor running on garbage):
    // last subframe's bookkeeping, then locate the CRC-16 footer.
    bool finished = false;
    auto finish_frame = [&]() {
        finished = true;
        if (L.status == CLX_OK) {
            if (L.pred && !L.params_done) parse_params(L);  // last subframe had order == block size
            if (L.status == CLX_OK && overrun(L)) L.status = CLX_ERR_IO_UNEXPECTED_EOF;
        }
        clx_frame_result res;
        res.status = L.status;
        res.consumed = 0;
        if (L.status == CLX_OK) {
            // Pad bits up to the byte boundary are skipped unchecked (src/frame.rs:744-750);
            // the CRC-16 footer must still be readable (:754).
            uint32_t end_bits = bc_pos(L.bc) - L.frame_bit0;
            uint32_t end_byte = (end_bits + 7) >> 3;
            if (end_byte + 2 > byte_len) res.status = CLX_ERR_IO_UNEXPECTED_EOF;
            res.consumed = end_byte + 2;
        }
        results[fidx] = res;
    };

    for (uint32_t it = 0; it < steps;) {
        // ------------------------------------------------------------------
        // events (rare, divergent): subframe boundaries, predictor parameters,
        // Rice partition boundaries
        // ------------------------------------------------------------------
        if (it < L.total) {
            if (L.mode != M_CONST || L.ch < L.nch) {
                if (L.t == L.bs && L.mode != M_HEADER) {  // subframe finished
                    if (L.pred && !L.params_done) parse_params(L);  // order == block size
                    if (L.ch < L.nch) { L.ch++; L.mode = M_HEADER; }
                }
                if (L.mode == M_HEADER) parse_subframe_header(L, need_hi);
                if (L.mode == M_VERB && L.pred && L.t == L.order) parse_params(L);
                if (L.mode == M_RICE && L.rem == 0 && L.parts_left > 0) {
                    next_partition(L, L.per);
                    if (L.mode == M_RICE && overrun(L)) fail(L, CLX_ERR_IO_UNEXPECTED_EOF);
                }
            }
        }
        if (have && !finished && it >= L.total) finish_frame();
        // How many steps can this lane run before its next event?
        uint32_t run;
        if (it >= L.total) run = 0xffffffffu;
        else if (L.mode == M_RICE) run = L.rem;
        else if (L.mode == M_VERB) run = (L.pred ? L.order : L.bs) - L.t;
        else run = (L.ch >= L.nch ? L.total - it : L.bs - L.t);  // constant subframe / zero fill
        uint32_t n = __reduce_min_sync(0xffffffffu, run);
        n = min(n, steps - it);
        const bool all_rice = __all_sync(0xffffffffu, it >= L.total || L.mode == M_RICE);
        const uint32_t ordmax = __reduce_max_sync(0xffffffffu, (it < L.total && L.mode == M_RICE) ? L.order : 0u);

        // ------------------------------------------------------------------
        // hot loop: every live lane is inside a Rice partition; 4 samples per trip
        // ------------------------------------------------------------------
        if (all_rice && (it & 3) == 0 && n >= 4) {
            uint32_t n4 = n & ~3u;
            const bool live = it < L.total;
            auto body = [&](auto taps_tag) {
                constexpr int TAPS = decltype(taps_tag)::value;
                for (uint32_t i = 0; i < n4; i += 4) {
                    int32_t v[KORD + 4];
#pragma unroll
                    for (int j = 0; j < KORD; j++) v[j] = L.h[j];
                    int32_t e0 = rice_decode(L);
                    int32_t e1 = rice_decode(L);
                    int32_t e2 = rice_decode(L);
                    int32_t e3 = rice_decode(L);
                    v[KORD + 0] = predict<KORD, TAPS>(v, 0, L.c, L.shift) + e0;
                    v[KORD + 1] = predict<KORD, TAPS>(v, 1, L.c, L.shift) + e1;
                    v[KORD + 2] = predict<KORD, TAPS>(v, 2, L.c, L.shift) + e2;
                    v[KORD + 3] = predict<KORD, TAPS>(v, 3, L.c, L.shift) + e3;
#pragma unroll
                    for (int j = KORD - TAPS; j < KORD; j++) L.h[j] = v[j + 4];
                    if (live) {
                        int4 o;
                        o.x = (int32_t)((uint32_t)v[KORD + 0] << L.wasted);
                        o.y = (int32_t)((uint32_t)v[KORD + 1] << L.wasted);
                        o.z = (int32_t)((uint32_t)v[KORD + 2] << L.wasted);
                        o.w = (int32_t)((uint32_t)v[KORD + 3] << L.wasted);
                        *reinterpret_cast<int4*>(tile + lane * 32 + ((((it >> 2) & 7) ^ (lane & 7)) << 2)) = o;
                    }
                    it += 4;
                    if ((it & 31) == 0) flush_tile(tile, rows, it - 32, lane);
                }
            };
            if (KORD > 12 && ordmax > 12) body(std::integral_constant<int, KORD>{});
            else if (ordmax > 8) body(std::integral_constant<int, (KORD < 12 ? KORD : 12)>{});
            else if (ordmax > 4) body(std::integral_constant<int, 8>{});
            else body(std::integral_constant<int, 4>{});
            if (live) { L.rem -= n4; L.t += n4; }
            continue;
        }

        // ------------------------------------------------------------------
        // generic steps: any mix of modes, one sample per trip
        // ------------------------------------------------------------------
        // (n >= 1 whenever events were processed to a fixpoint; never spin on a zero-length run)
        n = max(n, 1u);
        uint32_t ng = all_rice ? ((it & 3) ? min(n, 4 - (it & 3)) : min(n, 3u)) : n;
        for (uint32_t i = 0; i < ng; i++) {
            int32_t s = 0;
            const bool live = it < L.total;
            if (live) {
                if (L.mode == M_RICE) {
                    int32_t e = rice_decode(L);
                    long long acc = 0;
#pragma unroll
                    for (int j = 0; j < KORD; j++) acc += (long long)L.c[j] * (long long)L.h[j];
                    s = (int32_t)(acc >> L.shift) + e;
                    L.rem--;
                } else if (L.mode == M_VERB) {
                    s = hd_sext(bc_read(L.bc, L.sfbps), L.sfbps);
                } else {
                    s = L.cval;
                }
#pragma unroll
                for (int j = 0; j < KORD - 1; j++) L.h[j] = L.h[j + 1];
                L.h[KORD - 1] = s;
                L.t++;
                tile[tile_word(lane, it & 31)] = (int32_t)((uint32_t)s << L.wasted);
            }
            it++;
            if ((it & 31) == 0) flush_tile(tile, rows, it - 32, lane);
        }
    }
    // trailing partial tile
    if (steps & 31) flush_tile(tile, rows, steps & ~31u, lane);

    if (have && !finished) finish_frame();
}

// ---------------------------------------------------------------------------------
// launch
// ---------------------------------------------------------------------------------
cudaError_t launch_decode(const DecodeBuffers& b, const Plan& plan, bool crc, cudaStream_t stream, uint64_t* launches) {
    if (b.n_frames == 0) return cudaSuccess;
    const bool fast = plan.path != Path::Generic;
    // The lane-per-frame decode pass writes interleaved I32 / I16 and the channels modes itself when the caller keeps the
    // frames to convert after the generic kernel (`mark`); every other path, and I24, decodes to planar and converts all
    // frames at the end.
    const bool channels = b.mode == CLX_OUT_CHANNELS_I32 || b.mode == CLX_OUT_CHANNELS_F32;
    const bool fused = plan.path == Path::LanePerFrame && b.mark != nullptr &&
                       (b.mode == CLX_OUT_INTERLEAVED_I32 || b.mode == CLX_OUT_INTERLEAVED_I16 || channels);
    // planar -> the batch's mode, for the frames in `sel` (all if null) unless *gate == 0
    auto convert = [&](const uint8_t* sel, const int* gate) {
        return channels ? launch_channels(b.descs, b.n_frames, plan.max_frame_elems, b.out, b.conv, b.cols, b.stride, b.wins,
                                          b.mode, stream, launches, sel, gate)
                        : launch_interleave(b.descs, b.n_frames, plan.max_frame_elems, b.out, b.conv, b.mode, stream,
                                            launches, sel, gate);
    };
    int* d_generic = b.flags;        // set by a fast path: some frames need the generic kernel
    int* d_need_hi = b.flags + 1;    // set by the 12-tap generic instance: some frames need 32 taps
    int* d_need_wide = b.flags + 2;  // set by the lane-per-frame decode pass: some frames need the i64 second chance
    cudaError_t e = cudaMemsetAsync(b.flags, 0, 4 * sizeof(int), stream);
    if (e != cudaSuccess) return e;
    if (plan.path == Path::LanePerFrame)
        e = launch_seq(b.bytes, b.buf_bytes, b.descs, b.n_frames, fused ? static_cast<int32_t*>(b.conv) : b.out, b.results,
                       d_generic, d_need_wide, b.params, plan, fused ? b.mode : (uint32_t)CLX_OUT_PLANAR_I32, b.cols, b.stride,
                       b.wins, stream, launches);
    else if (plan.path == Path::WarpPerFrame)
        e = launch_warp_per_frame(b.bytes, b.buf_bytes, b.descs, b.n_frames, b.out, b.results, d_generic, b.params, plan,
                                  stream, launches);
    if (e != cudaSuccess) return e;
    if (!(fast && plan.no_generic)) {  // (testing: no_generic leaves the fast path's verdicts as they are)
        if (fused) {  // the frames the generic kernel is about to take over, whatever the fast path wrote for them
            e = launch_mark_status(b.results, b.n_frames, CLX_INTERNAL_NEED_GENERIC, b.mark, d_generic, stream, launches);
            if (e != cudaSuccess) return e;
        }
        const uint32_t per_cta = WARPS_PER_CTA * 32;
        dim3 grid((b.n_frames + per_cta - 1) / per_cta), block(per_cta);
        // After a fast path: only the frames it declined, and nothing at all when it declined none.
        decode_frames_kernel<12><<<grid, block, 0, stream>>>(b.bytes, b.buf_bytes, b.descs, b.n_frames, b.out, b.results,
                                                             d_need_hi, fast ? d_generic : nullptr,
                                                             fast ? CLX_INTERNAL_NEED_GENERIC : 0);
        (*launches)++;
        // Frames with an LPC order above 12 (non-subset streams) were only flagged by the 12-tap
        // instance; the 32-tap instance picks them up.  It exits immediately when nothing was flagged.
        decode_frames_kernel<32><<<grid, block, 0, stream>>>(b.bytes, b.buf_bytes, b.descs, b.n_frames, b.out, b.results,
                                                             d_need_hi, d_need_hi, CLX_INTERNAL_NEED_HIGH_ORDER);
        (*launches)++;
        if (fused) {
            // The marked frames' planar samples -> the batch's mode, over every element of each: nothing the fast path
            // wrote for them survives.  Gated like the 12-tap instance: exits at once when the fast path declined nothing.
            e = convert(b.mark, d_generic);
            if (e != cudaSuccess) return e;
        }
    }
    if (crc) {  // src/frame.rs:752-763, after the subframes
        e = launch_crc16(b.bytes, b.descs, b.n_frames, b.results, stream, launches);
        if (e != cudaSuccess) return e;
    }
    if (b.mode != CLX_OUT_PLANAR_I32 && !fused) {
        e = convert(nullptr, nullptr);
        if (e != cudaSuccess) return e;
    }
    return cudaGetLastError();
}

}  // namespace clx
