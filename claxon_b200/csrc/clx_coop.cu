// clx_coop.cu — the fast path of claxon_b200: warp-cooperative entropy decode + lane-per-subframe
// prediction, as two kernels working in place on the output buffer.
//
//   1. `entropy_frames_kernel` — ONE WARP PER FRAME.  The warp walks its frame's bitstream — subframe
//      header, warm-up samples, LPC parameters, residual header, Rice partitions (reference
//      src/subframe.rs:29-91, :236-380, :382-415, :651-701) — and decodes the Rice residuals of a
//      partition 4096 bits at a time with all 32 lanes: every lane owns four 32-bit words of the
//      window and walks them simultaneously for the *speculated* code phase ("a search for the next
//      unary terminator starts at bit 0 of every word"); a shuffle fix-point then makes the phases
//      exact — a word's entry phase is its left neighbour's exit phase, and a re-walk from a
//      corrected phase stops as soon as it meets a terminator of the speculated chain, from where
//      both coincide; popcount + shuffle prefix sums rank the codes, a shuffle max-scan gives every
//      code the end of its predecessor (hence its unary quotient), and each lane emits its codes
//      (rice_to_signed, src/subframe.rs:157-170) at their final position in the frame's output
//      block.  Residuals, warm-up, verbatim and constant samples therefore already sit where the PCM
//      will be; predictor parameters go to a small per-subframe table.
//   2. `predict_frames_kernel` — ONE LANE PER SUBFRAME.  predict_fixed / predict_lpc_* (src/subframe.rs:
//      417-474, :524-614) are strictly serial recurrences — the floor in `>> qlp_shift` makes them
//      non-associative — so the parallel axis is the set of subframes: 32 of them advance per warp
//      instruction, coefficients and history register-resident, residuals streamed from the output
//      block with 16-byte loads two trips ahead.  Wasted-bits shift (src/subframe.rs:216-225) and
//      inter-channel decorrelation (src/frame.rs:319-389, partner channel = neighbouring lane, one
//      shuffle) happen in registers; samples leave through a swizzled 32x32 shared-memory transpose
//      as coalesced 16-byte stores, over the residuals they replace (the two kernels run back to back,
//      so when a batch's output fits the 50 MB L2 of an H100 — a 1024-frame C2 batch writes 34 MB —
//      its residuals are read back from L2).
//
// Anything this path does not handle exactly — malformed input of any kind, the Rice escape code,
// unary runs longer than a window, more than 8 channels — is not guessed at: the frame is flagged
// and the generic lane-per-frame kernel (clx_decode.cu), which reproduces claxon's error precedence,
// decodes it afterwards.
#include <cuda_runtime.h>
#include <stdint.h>

#include "claxon_b200.h"
#include <algorithm>
#include <cstdlib>

#include "clx_internal.h"
#include "clx_lanes.h"

namespace clx {

struct SubParams {   // one per subframe (global memory, written by the entropy kernel)
    int32_t order;   // predictor order; 0 = nothing to predict (constant / verbatim / fixed-0)
    int32_t shift;   // qlp shift (0 for fixed predictors)
    int32_t wasted;  // wasted bits per sample
    uint32_t narrow; // 0: predicted with the i64 accumulator; else sum|coef| of a subframe predicted with
                     // the i32 accumulator (phase 3 verifies that this was exact)
    int16_t coefs[32];  // coefs[j] multiplies s[t-1-j]
};


// ---------------------------------------------------------------------------------
// Warp-wide bit window: 256 consecutive big-endian words of the frame, 16-byte aligned.
// Lane l holds words 4l..4l+3 of the current 128-word window in X (byte-swapped, ready for bit
// arithmetic) and the same slice of the NEXT window in Y, raw as loaded: Y is fetched one window
// ahead with a single coalesced 16-byte load per lane and nothing touches it until it slides into
// X, so HBM/L2 latency stays off the critical path.  All field extraction is shuffle + funnel shift.
// ---------------------------------------------------------------------------------
constexpr uint32_t WPL = 4;            // words per lane
constexpr uint32_t STAGE_CODES = 1024;  // codes one window may emit (a window with more is cut short)
constexpr uint32_t WIN_WORDS = 32 * WPL;

struct Win {
    const uint4* base;  // 16-byte aligned global address at or before the frame's first byte
    uint32_t qlim;      // first 16-byte group index that lies outside the byte buffer (reads give 0)
    uint32_t b0;        // word index (multiple of 4) of X[0] of lane 0
    uint32_t X[WPL], Y[WPL];
    uint32_t F[WPL];    // words loaded by the previous slide, not yet merged into Y (pending != 0)
    uint32_t pending;
};

__device__ __forceinline__ uint4 win_ldg(const Win& w, uint32_t quad) {
    uint4 v = make_uint4(0, 0, 0, 0);
    if (quad < w.qlim) v = __ldg(w.base + quad);
    return v;
}
__device__ __forceinline__ void win_prime(Win& w, uint32_t bitpos, uint32_t lane) {
    w.b0 = (bitpos >> 5) & ~3u;
    const uint4 x = win_ldg(w, (w.b0 >> 2) + lane), y = win_ldg(w, (w.b0 >> 2) + 32 + lane);
    w.X[0] = hd_bswap(x.x); w.X[1] = hd_bswap(x.y); w.X[2] = hd_bswap(x.z); w.X[3] = hd_bswap(x.w);
    w.Y[0] = y.x; w.Y[1] = y.y; w.Y[2] = y.z; w.Y[3] = y.w;
    w.pending = 0;
}
// Slides the window so that the 16-byte group containing `bitpos` is lane 0's.
__device__ __forceinline__ void win_advance(Win& w, uint32_t bitpos, uint32_t lane) {
    const uint32_t nb0 = (bitpos >> 5) & ~3u;
    const uint32_t d = (nb0 - w.b0) >> 2;  // lanes to shift by
    if (d == 0) return;
    if (d > 32) { win_prime(w, bitpos, lane); return; }
    // The words fetched by the previous slide are only now folded into Y: a register written by a
    // load is not touched until a whole window later, so the load's latency is never waited for.
    if (w.pending) {
#pragma unroll
        for (uint32_t j = 0; j < WPL; j++) w.Y[j] = w.F[j];
    }
    const uint32_t src = (lane + d) & 31;
    const bool low = lane + d < 32;
    w.b0 = nb0;
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) {
        const uint32_t xs = __shfl_sync(0xffffffffu, w.X[j], src);
        const uint32_t ys = __shfl_sync(0xffffffffu, w.Y[j], src);
        w.X[j] = low ? xs : hd_bswap(ys);
        w.Y[j] = ys;  // lanes with !low get their real Y from F at the next slide
    }
    w.pending = low ? 0u : 1u;
    if (!low) {
        const uint4 fresh = win_ldg(w, (nb0 >> 2) + 32 + lane);
        w.F[0] = fresh.x; w.F[1] = fresh.y; w.F[2] = fresh.z; w.F[3] = fresh.w;
    }
}
// Word `i` (0 .. WIN_WORDS-1, uniform across the warp) of the window.
__device__ __forceinline__ uint32_t win_word(const Win& w, uint32_t i) {
    const uint32_t j = i & 3;
    const uint32_t mine = j == 0 ? w.X[0] : j == 1 ? w.X[1] : j == 2 ? w.X[2] : w.X[3];
    return __shfl_sync(0xffffffffu, mine, (i >> 2) & 31);
}
// 32 bits starting at `bitpos` (uniform); requires the word of bitpos to be at most WIN_WORDS-2.
__device__ __forceinline__ uint32_t win_peek32(const Win& w, uint32_t bitpos) {
    const uint32_t i = (bitpos >> 5) - w.b0;
    return __funnelshift_l(win_word(w, i + 1), win_word(w, i), bitpos & 31);
}
__device__ __forceinline__ uint32_t top_bits(uint32_t v, uint32_t n) {  // n in [0,32]
    return n >= 32 ? v : __funnelshift_l(v, 0, n);
}
// Per-lane variant: every lane asks for its own bit position inside the window.
__device__ __forceinline__ uint32_t win_peek32_lane(const Win& w, uint32_t bitpos) {
    const uint32_t i = (bitpos >> 5) - w.b0, i1 = i + 1;
    uint32_t a[WPL], b[WPL];
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) {
        a[j] = __shfl_sync(0xffffffffu, w.X[j], (i >> 2) & 31);
        b[j] = __shfl_sync(0xffffffffu, w.X[j], (i1 >> 2) & 31);
    }
    const uint32_t w0 = (i & 3) == 0 ? a[0] : (i & 3) == 1 ? a[1] : (i & 3) == 2 ? a[2] : a[3];
    const uint32_t w1 = (i1 & 3) == 0 ? b[0] : (i1 & 3) == 1 ? b[1] : (i1 & 3) == 2 ? b[2] : b[3];
    return __funnelshift_l(w1, w0, bitpos & 31);
}

// ---------------------------------------------------------------------------------
// Rice decode of one window.  Vocabulary: a *search* looks for the next unary terminator (a 1 bit)
// from some bit offset; after a terminator at t the next search starts at t+1+k.  The *phase* of a
// lane is the offset (into its first word) at which the first search inside its 128-bit span
// starts; walking the span from a phase yields the terminator masks of its words and the exit phase
// (the next lane's entry phase).
//
// Every lane first walks its span for the *speculated* phase 0.  A shuffle fix-point then makes the
// phases exact: a lane whose entry phase turns out different re-walks, but only until it meets a
// terminator of its own speculated chain — from there on both chains coincide — so a correction
// costs a couple of codes, and since 128 bits hold many codes almost every re-walk does merge and
// the fix-point settles in one or two rounds.
// ---------------------------------------------------------------------------------
struct LaneWalk {
    uint32_t tm[WPL];  // terminator masks (bit 31 = first bit of the word)
    uint32_t x;        // exit phase
};

// Walks the lane's words from word `j0`, phase `e`.  When `merge`, stops at the first terminator
// shared with the speculated walk and adopts its remainder.
__device__ __forceinline__ void walk_lane(const uint32_t (&W)[WPL], uint32_t j0, uint32_t e, uint32_t k, bool merge,
                                          const LaneWalk& spec, LaneWalk& out) {
    uint32_t o = e;
    bool merged = false;
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) {
        uint32_t tm = 0;
        if (merged) tm = spec.tm[j];
        else if (j >= j0) {
            while (o < 32) {
                const uint32_t m = W[j] & (0xffffffffu >> o);
                if (m == 0) { o = 32; break; }  // the search carries on in the next word, phase 0
                const uint32_t t = __clz(m);
                const uint32_t bit = 0x80000000u >> t;
                if (merge && (spec.tm[j] & bit)) {
                    tm |= spec.tm[j] & (bit | (bit - 1));
                    merged = true;
                    break;
                }
                tm |= bit;
                o = t + 1 + k;
            }
            if (!merged) o -= 32;
        }
        out.tm[j] = tm;
    }
    out.x = merged ? spec.x : o;
}

// Decodes up to `n_rem` Rice codes with parameter k starting at bit `P` from the current window
// into out[0..); returns the number decoded (0 = cannot make progress here) and advances P to
// the end of the last decoded code.  The very last word of the window is never owned (it only
// lends its bits as the right-hand neighbour), so Y is not read here.
__device__ __forceinline__ uint32_t rice_window(const Win& w, uint32_t& P, uint32_t k, uint32_t n_rem, int32_t* out,
                                                int32_t* stage, uint32_t lane) {
    n_rem = min(n_rem, STAGE_CODES);
    const uint32_t s = P - (w.b0 << 5);      // < 128: where the first search starts
    const uint32_t first = s >> 5;           // lane 0's word that contains it
    uint32_t W[WPL], WN[WPL];
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) W[j] = w.X[j];
    const uint32_t right = __shfl_down_sync(0xffffffffu, w.X[0], 1);
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) WN[j] = j + 1 < WPL ? w.X[j + 1] : right;
    if (lane == 31) W[WPL - 1] = 0;  // lent only: no terminators of its own

    // 1. speculated walk: phase 0 (lane 0 knows its true start)
    LaneWalk spec, cur;
    const uint32_t j0 = lane == 0 ? first : 0u;
    uint32_t e = lane == 0 ? (s & 31u) : 0u;
    walk_lane(W, j0, e, k, false, spec, spec);
    cur = spec;
    // 2. fix-point on the entry phases
    for (;;) {
        const uint32_t left = __shfl_up_sync(0xffffffffu, cur.x, 1);
        const bool redo = lane > 0 && left != e;
        if (!__any_sync(0xffffffffu, redo)) break;
        if (redo) {
            e = left;
            walk_lane(W, 0, e, k, true, spec, cur);
        }
    }
    // 3. ranks
    uint32_t cnt[WPL], lane_cnt = 0;
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) { cnt[j] = __popc(cur.tm[j]); lane_cnt += cnt[j]; }
    uint32_t incl = lane_cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (uint32_t)d) incl += v;
    }
    uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t rank[WPL];
    rank[0] = incl - lane_cnt;
#pragma unroll
    for (uint32_t j = 1; j < WPL; j++) rank[j] = rank[j - 1] + cnt[j - 1];
    if (total > n_rem) {  // the partition ends inside this window: keep the first n_rem codes
#pragma unroll
        for (uint32_t j = 0; j < WPL; j++) {
            if (rank[j] >= n_rem) cur.tm[j] = 0;
            else if (rank[j] + cnt[j] > n_rem) {
                uint32_t keep = 0, tmp = cur.tm[j];
                for (uint32_t i = 0; i < n_rem - rank[j]; i++) {
                    const uint32_t bit = 0x80000000u >> __clz(tmp);
                    keep |= bit;
                    tmp &= ~bit;
                }
                cur.tm[j] = keep;
            }
        }
        total = n_rem;
    }
    if (total == 0) return 0;
    // 4. end of the last code at or before each lane (window-relative bit offsets)
    uint32_t lane_end = 0;
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++)
        if (cur.tm[j]) lane_end = ((lane * WPL + j) << 5) + (32 - __ffs(cur.tm[j])) + 1 + k;
    uint32_t endi = lane_end;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, endi, d);
        if (lane >= (uint32_t)d) endi = max(endi, v);
    }
    uint32_t start = __shfl_up_sync(0xffffffffu, endi, 1);
    if (lane == 0) start = 0;
    start = max(start, s);
    const uint32_t new_end = __shfl_sync(0xffffffffu, endi, 31);
    // 5. emit, word after word, into the warp's staging buffer.  A lane's codes are consecutive in
    // the output but 32 lanes' stores would touch 32 different sectors; staged, the window leaves
    // as full 16-byte vectors.  Staging index and global element index agree modulo 4.
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(out) >> 2) & 3u;
    uint32_t idx = mis + rank[0];
#pragma unroll
    for (uint32_t j = 0; j < WPL; j++) {
        uint32_t rest = cur.tm[j];
        while (rest) {
            const uint32_t t = __clz(rest);
            rest &= ~(0x80000000u >> t);
            const uint32_t pos = ((lane * WPL + j) << 5) + t;
            const uint32_t q = pos - start;
            const uint32_t hi = __funnelshift_lc(WN[j], W[j], t + 1);
            const uint32_t r = __funnelshift_l(hi, 0, k);
            const uint32_t u = (q << k) | r;
            stage[idx++] = (int32_t)((u >> 1) ^ (0u - (u & 1u)));
            start = pos + 1 + k;
        }
    }
    __syncwarp();
    // 6. flush: group g holds staging words [4g, 4g+4) = output elements [4g - mis, 4g - mis + 4)
    const uint32_t hi_idx = mis + total;
    for (uint32_t g4 = lane * 4; g4 < hi_idx; g4 += 128) {
        const int4 v = *reinterpret_cast<const int4*>(stage + g4);
        int32_t* dst = out + g4 - mis;   // 16-byte aligned by construction
        if (g4 >= mis && g4 + 4 <= hi_idx) *reinterpret_cast<int4*>(dst) = v;
        else {
            if (g4 >= mis && g4 < hi_idx) dst[0] = v.x;
            if (g4 + 1 >= mis && g4 + 1 < hi_idx) dst[1] = v.y;
            if (g4 + 2 >= mis && g4 + 2 < hi_idx) dst[2] = v.z;
            if (g4 + 3 < hi_idx) dst[3] = v.w;
        }
    }
    __syncwarp();
    P = (w.b0 << 5) + new_end;
    return total;
}

// Per-lane, branch-free form for the predict kernel: the lane holds one channel's sample `own`, its
// neighbour's is `other`.  Every case of src/frame.rs:319-389 is (own*p + other*q + side&1) >> s in
// wrapping i32 with per-lane constants (side = channel 1's sample):
//   independent      p= 1 q=0            left/side  ch0: p=1 q=0    ch1 (left - side): p=-1 q=1
//   side/right ch0 (side + right): p=1 q=1   ch1: p=1 q=0
//   mid/side   ch0: (2*mid + (side&1) + side) >> 1 : p=2 q=1, bit from other
//              ch1: (2*mid + (side&1) - side) >> 1 : p=-1 q=2, bit from own
struct DecorLane { uint32_t p, q, own_bit, other_bit, s; };
__device__ __forceinline__ DecorLane decor_consts(uint32_t ca, bool second) {
    DecorLane d = {1u, 0u, 0u, 0u, 0u};
    if (ca == 8 && second) { d.p = 0xffffffffu; d.q = 1u; }
    else if (ca == 9 && !second) { d.q = 1u; }
    else if (ca == 10) {
        d.s = 1u;
        if (second) { d.p = 0xffffffffu; d.q = 2u; d.own_bit = 1u; }
        else { d.p = 2u; d.q = 1u; d.other_bit = 1u; }
    }
    return d;
}
__device__ __forceinline__ int32_t decor_lane(uint32_t own, uint32_t other, const DecorLane& d) {
    const uint32_t t = own * d.p + other * d.q + (own & d.own_bit) + (other & d.other_bit);
    return ((int32_t)t) >> d.s;
}

constexpr int ENT_WARPS = 4;   // entropy kernel: frames (warps) per CTA
constexpr int PRE_WARPS = 2;   // predict kernel: warps per CTA
constexpr int RING_SAMPLES = 64;                 // predict kernel: residual ring per lane
constexpr int RING_LANE_WORDS = RING_SAMPLES + 4; // +16 bytes of skew: 16-byte accesses of 8 lanes hit 32 banks

// ---------------------------------------------------------------------------------
// Kernel 1: entropy decode, one warp per frame, output block written in place
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(ENT_WARPS * 32)
entropy_frames_kernel(const uint8_t* __restrict__ bytes, uint64_t buf_bytes, const clx_frame_desc* __restrict__ descs,
                      uint32_t n_frames, int32_t* __restrict__ out, clx_frame_result* __restrict__ results,
                      SubParams* __restrict__ params, uint32_t CH, int* __restrict__ need_generic) {
    __shared__ __align__(16) int32_t s_stage[ENT_WARPS][STAGE_CODES + 4];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t fidx = blockIdx.x * ENT_WARPS + warp;
    if (fidx >= n_frames) return;
    int32_t* stage = s_stage[warp];
    const clx_frame_desc d = descs[fidx];
    const uint32_t bs = d.block_size, nch = d.n_channels, ca = d.channel_assignment;
    bool ok = nch <= CH && d.bits_per_sample != 0;
    int32_t* fbuf = out + d.out_offset;
    Win w;
    const uint64_t aligned = d.byte_offset & ~15ull;
    w.base = reinterpret_cast<const uint4*>(bytes + aligned);
    w.qlim = (uint32_t)min((buf_bytes - aligned) >> 4, (uint64_t)0x7ffffffu);
    const uint32_t bit0 = (uint32_t)(d.byte_offset & 15) * 8;
    const uint32_t limit = bit0 + d.byte_len * 8;
    uint32_t P = bit0 + (uint32_t)d.header_len * 8;
    win_prime(w, P, lane);

    for (uint32_t ch = 0; ok && ch < nch; ch++) {
        uint32_t bps = d.bits_per_sample;
        if (ca == 9) bps += (ch == 0);                 // side/right: side first (src/frame.rs:725)
        else if (ca == 8 || ca == 10) bps += (ch == 1);  // src/frame.rs:717, :736
        int32_t* sbuf = fbuf + (size_t)ch * bs;
        SubParams* sp = params + (size_t)fidx * CH + ch;
        win_advance(w, P, lane);
        // ---- subframe header (src/subframe.rs:29-91) ----
        const uint32_t head = win_peek32(w, P) >> 24;
        P += 8;
        if (head & 0x80u) { ok = false; break; }
        const uint32_t code = (head >> 1) & 0x3fu;
        uint32_t order = 0;
        int type;
        if (code == 0) type = 0;
        else if (code == 1) type = 1;
        else if ((code & 0x3eu) == 0x02u || (code & 0x3cu) == 0x04u || (code & 0x30u) == 0x10u) { ok = false; break; }
        else if ((code & 0x38u) == 0x08u) { order = code & 7u; if (order > 4) { ok = false; break; } type = 2; }
        else { order = (code & 0x1fu) + 1; type = 3; }
        uint32_t wasted = 0;
        if (head & 1u) {
            const uint32_t v = win_peek32(w, P);
            if (v == 0) { ok = false; break; }  // > 31 wasted bits: an error for the generic kernel to name
            const uint32_t q = __clz(v);
            wasted = q + 1;
            P += q + 1;
        }
        if (wasted >= bps) { ok = false; break; }
        const uint32_t sfbps = bps - wasted;
        if (sfbps > 30) { ok = false; break; }
        if ((type == 2 || type == 3) && order > bs) { ok = false; break; }
        if (lane == 0) { sp->order = 0; sp->shift = 0; sp->wasted = (int32_t)wasted; sp->narrow = 0; }
        if (type == 0) {  // constant (src/subframe.rs:382-394)
            const int32_t v = hd_sext(top_bits(win_peek32(w, P), sfbps), sfbps);
            P += sfbps;
            for (uint32_t i = lane; i < bs; i += 32) sbuf[i] = v;
            if (P > limit) { ok = false; break; }
            continue;
        }
        // ---- verbatim samples: the whole subframe, or the warm-up (src/subframe.rs:397-415) ----
        const uint32_t n_raw = type == 1 ? bs : order;
        for (uint32_t i0 = 0; i0 < n_raw; i0 += 32) {
            win_advance(w, P, lane);
            const uint32_t i = i0 + lane;
            const uint32_t v = win_peek32_lane(w, P + lane * sfbps);
            if (i < n_raw) sbuf[i] = hd_sext(top_bits(v, sfbps), sfbps);
            P += min(32u, n_raw - i0) * sfbps;
        }
        if (P > limit) { ok = false; break; }
        if (type == 1) continue;
        // ---- predictor parameters (src/subframe.rs:427-431, :669-701) ----
        win_advance(w, P, lane);
        uint32_t shift = 0;
        if (type == 3) {
            const uint32_t pq = win_peek32(w, P) >> 23;  // 4-bit precision-1, 5-bit signed shift
            P += 9;
            const uint32_t prec_m1 = pq >> 5;
            if (prec_m1 == 15) { ok = false; break; }
            const uint32_t precision = prec_m1 + 1;
            const int32_t sh = hd_sext(pq & 31u, 5);
            if (sh < 0) { ok = false; break; }
            shift = (uint32_t)sh;
            const uint32_t v = win_peek32_lane(w, P + lane * precision);
            if (lane < order) sp->coefs[lane] = (int16_t)hd_sext(top_bits(v, precision), precision);
            P += order * precision;
        } else if (lane < 4) {
            sp->coefs[lane] = (int16_t)(int8_t)(fixed_coefs_packed(order) >> (8 * lane));
        }
        if (lane == 0) { sp->order = (int32_t)order; sp->shift = (int32_t)shift; }
        // ---- residual (src/subframe.rs:236-380) ----
        win_advance(w, P, lane);
        const uint32_t rh = win_peek32(w, P) >> 26;  // 2-bit coding method, 4-bit partition order
        P += 6;
        const uint32_t method = rh >> 4, po = rh & 15u;
        if (method > 1) { ok = false; break; }
        const uint32_t n_part = 1u << po;
        if ((bs & ((n_part - 1u) & 0xffffu)) != 0) { ok = false; break; }
        const uint32_t per = bs >> po;
        if (order > per) { ok = false; break; }
        const uint32_t pbits = method == 0 ? 4u : 5u;
        uint32_t at = order;
        for (uint32_t part = 0; ok && part < n_part; part++) {
            win_advance(w, P, lane);
            const uint32_t k = win_peek32(w, P) >> (32 - pbits);
            P += pbits;
            if (k == (1u << pbits) - 1u) { ok = false; break; }  // escape code: Unsupported in the reference
            uint32_t n_rem = part == 0 ? per - order : per;
            while (n_rem > 0) {
                win_advance(w, P, lane);
                const uint32_t got = rice_window(w, P, k, n_rem, sbuf + at, stage, lane);
                if (got == 0 || P > limit) { ok = false; break; }
                at += got;
                n_rem -= got;
            }
        }
        if (P > limit) ok = false;
    }
    // frame footer: pad to the byte boundary, the CRC-16 must be readable (src/frame.rs:744-754)
    uint32_t consumed = 0;
    if (ok) {
        const uint32_t end_byte = (P - bit0 + 7) >> 3;
        consumed = end_byte + 2;
        if (P > limit || consumed > d.byte_len) ok = false;
    }
    if (lane == 0) {
        clx_frame_result res;
        res.status = ok ? (int32_t)CLX_OK : (int32_t)CLX_INTERNAL_NEED_GENERIC;
        res.consumed = consumed;
        results[fidx] = res;
        if (!ok) *need_generic = 1;
    }
}

// ---------------------------------------------------------------------------------
// Kernel 2: prediction + wasted shift + decorrelation, one lane per subframe, in place
// ---------------------------------------------------------------------------------
struct PredRow {       // per lane, shared memory: where the lane's samples go
    int32_t* out;      // subframe's first output element (nullptr: idle lane)
    uint32_t bs;       // block size
    uint32_t vec_ok;   // 16-byte stores allowed
};

// Writes the warp's 32x32 tile (steps [g0, g0+32) of every lane's subframe) to global memory.
__device__ __forceinline__ void flush_rows(const int32_t* tile, const PredRow* rows, uint32_t g0, uint32_t lane) {
    __syncwarp();
#pragma unroll 2
    for (uint32_t pass = 0; pass < 8; pass++) {
        const uint32_t r = pass * 4 + (lane >> 3), grp = lane & 7;
        const PredRow pr = rows[r];
        const uint32_t g = g0 + grp * 4;
        if (pr.out != nullptr && g < pr.bs) {
            const int4 v = *reinterpret_cast<const int4*>(tile + r * 32 + ((grp ^ (r & 7)) << 2));
            if (pr.vec_ok && g + 4 <= pr.bs) *reinterpret_cast<int4*>(pr.out + g) = v;
            else {
                pr.out[g] = v.x;
                if (g + 1 < pr.bs) pr.out[g + 1] = v.y;
                if (g + 2 < pr.bs) pr.out[g + 2] = v.z;
                if (g + 3 < pr.bs) pr.out[g + 3] = v.w;
            }
        }
    }
    __syncwarp();
}

template <int TAPS, int U, typename ACC>
__device__ __forceinline__ void predict_rows(const int32_t* __restrict__ src, uint32_t bs, uint32_t order, uint32_t shift,
                                             uint32_t wasted, uint32_t ca, bool second, const int16_t* coefs, bool active,
                                             int32_t* tile, const PredRow* rows, int32_t* ring, uint32_t lane, int32_t& smin,
                                             int32_t& smax) {
    int32_t c[TAPS], h[TAPS];  // c[j] multiplies s[t-1-j]; h[j] = s[t-1-j]
#pragma unroll
    for (int j = 0; j < TAPS; j++) {
        c[j] = (active && (uint32_t)j < order) ? (int32_t)coefs[j] : 0;
        // Opaque to the optimiser: otherwise the i16 -> i64 promotion is folded into a full 64-bit
        // multiply (3 instructions) instead of one signed 32x32+64 IMAD.WIDE per tap.
        asm volatile("" : "+r"(c[j]));
        h[j] = 0;
    }
    const uint32_t max_bs = __reduce_max_sync(0xffffffffu, active ? bs : 0u);
    const uint32_t min_bs = __reduce_min_sync(0xffffffffu, active ? bs : 0xffffffffu);
    const uint32_t max_order = __reduce_max_sync(0xffffffffu, active ? order : 0u);
    const bool aligned = __all_sync(0xffffffffu, !active || ((reinterpret_cast<uintptr_t>(src) & 15) == 0));
    const uint32_t head_end = min(max_bs, (max_order + 31u) & ~31u);  // whole tiles
    const uint32_t bulk_end = (aligned && min_bs > head_end) ? head_end + ((min_bs - head_end) & ~31u) : head_end;

    // emits one finished sample of every lane: wasted shift, decorrelation with the neighbouring lane,
    // staging into the transpose tile, flush every 32 steps
    const DecorLane dl = decor_consts(ca, second);
    auto emit = [&](uint32_t t, int32_t s) {
        int32_t o = (int32_t)((uint32_t)s << wasted);
        const int32_t partner = __shfl_xor_sync(0xffffffffu, o, 1);
        o = decor_lane((uint32_t)o, (uint32_t)partner, dl);
        tile[tile_word(lane, t & 31)] = o;
        if ((t & 31) == 31) flush_rows(tile, rows, t - 31, lane);
    };
    auto guarded = [&](uint32_t t0, uint32_t t1) {  // one sample at a time, every condition checked
        for (uint32_t t = t0; t < t1; t++) {
            const bool inside = active && t < bs;
            int32_t val = inside ? src[t] : 0;
            if (t >= order) {
                long long acc = 0;
#pragma unroll
                for (int j = 0; j < TAPS; j++) acc += (long long)c[j] * (long long)h[j];
                val += sizeof(ACC) == 8 ? (int32_t)(acc >> shift) : (int32_t)((int32_t)acc >> shift);
            }
#pragma unroll
            for (int j = TAPS - 1; j > 0; j--) h[j] = h[j - 1];
            h[0] = val;
            if (inside) { smin = min(smin, val); smax = max(smax, val); }
            emit(t, val);
        }
    };
    guarded(0, head_end);
    if (bulk_end > head_end) {
        int32_t v[TAPS + U];
#pragma unroll
        for (int j = 0; j < TAPS; j++) v[j] = h[TAPS - 1 - j];
        // Residuals stream HBM/L2 -> shared memory through a per-lane ring filled by cp.async
        // (LDGSTS, 16 bytes per copy) DEPTH trips ahead of their use, so neither DRAM nor L2 latency
        // is ever waited for; idle lanes copy some active lane's data and ignore it.
        constexpr int Q = U / 4;                 // 16-byte copies per trip
        constexpr int SLOTS = RING_SAMPLES / U;  // trips the ring holds
        constexpr int DEPTH = SLOTS - 2;         // trips in flight
        const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(ring);
        auto request = [&](uint32_t trip) {      // trip index relative to head_end
            const uint32_t t = min(head_end + trip * U, bulk_end - U);
#pragma unroll
            for (int q = 0; q < Q; q++)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(ring_s + ((trip % SLOTS) * U + 4 * q) * 4),
                             "l"(src + t + 4 * q));
            asm volatile("cp.async.commit_group;");
        };
#pragma unroll
        for (int p = 0; p < DEPTH; p++) request(p);
        uint32_t trip = 0;
        for (uint32_t t = head_end; t < bulk_end; t += U, trip++) {
            request(trip + DEPTH);
            asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH));
            int32_t r[U];
#pragma unroll
            for (int q = 0; q < Q; q++) {
                const int4 x = *reinterpret_cast<const int4*>(ring + (trip % SLOTS) * U + 4 * q);
                r[4 * q] = x.x; r[4 * q + 1] = x.y; r[4 * q + 2] = x.z; r[4 * q + 3] = x.w;
            }
            seq_trip<TAPS, U, ACC>(v, c, r, shift);
#pragma unroll
            for (int i = 0; i < U; i++) {
                smin = min(smin, v[TAPS + i]);
                smax = max(smax, v[TAPS + i]);
            }
            // wasted shift + decorrelation + staging, 4 samples per 16-byte shared store
#pragma unroll
            for (int q = 0; q < Q; q++) {
                int32_t o[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    o[i] = (int32_t)((uint32_t)v[TAPS + 4 * q + i] << wasted);
                    const int32_t partner = __shfl_xor_sync(0xffffffffu, o[i], 1);
                    o[i] = decor_lane((uint32_t)o[i], (uint32_t)partner, dl);
                }
                const uint32_t col = (t + 4 * q) & 31;
                *reinterpret_cast<int4*>(tile + lane * 32 + (((col >> 2) ^ (lane & 7)) << 2)) = make_int4(o[0], o[1], o[2], o[3]);
            }
            if (((t + U) & 31) == 0) flush_rows(tile, rows, t + U - 32, lane);
#pragma unroll
            for (int j = 0; j < TAPS; j++) v[j] = v[j + U];
        }
#pragma unroll
        for (int j = 0; j < TAPS; j++) h[j] = v[TAPS - 1 - j];
        asm volatile("cp.async.wait_group 0;");  // the look-ahead copies past the bulk are never used
    }
    guarded(bulk_end, max_bs);
    if (max_bs & 31) flush_rows(tile, rows, max_bs & ~31u, lane);
}

__global__ void __launch_bounds__(PRE_WARPS * 32)
predict_frames_kernel(const clx_frame_desc* __restrict__ descs, uint32_t n_frames, int32_t* __restrict__ out,
                      clx_frame_result* __restrict__ results, const SubParams* __restrict__ params, uint32_t CH,
                      int* __restrict__ need_generic) {
    __shared__ __align__(16) int32_t s_tile[PRE_WARPS][32 * 32];
    __shared__ __align__(16) PredRow s_rows[PRE_WARPS][32];
    __shared__ __align__(16) int32_t s_ring[PRE_WARPS][32 * RING_LANE_WORDS];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t slot = (blockIdx.x * PRE_WARPS + warp) * 32 + lane;  // CH is a power of two: frames never split
    const uint32_t f = slot / CH, c = slot % CH;
    int32_t* tile = s_tile[warp];
    PredRow* rows = s_rows[warp];

    bool active = false, narrow_ok = true, second = false;
    uint32_t bs = 0, order = 0, shift = 0, wasted = 0, ca = 0, absum = 0;
    const int16_t* coefs = params[0].coefs;
    int32_t* sub = out;
    if (f < n_frames && results[f].status == CLX_OK) {
        const clx_frame_desc d = descs[f];
        if (c < d.n_channels) {
            const SubParams* sp = params + (size_t)f * CH + c;
            active = true;
            bs = d.block_size;
            order = (uint32_t)sp->order;
            shift = (uint32_t)sp->shift;
            wasted = (uint32_t)sp->wasted;
            coefs = sp->coefs;
            ca = d.channel_assignment >= 8 ? d.channel_assignment : 0u;
            second = c == 1;
            sub = out + d.out_offset + (size_t)c * bs;
            for (uint32_t j = 0; j < order; j++) absum += (uint32_t)abs((int)coefs[j]);
            uint32_t bits = d.bits_per_sample;  // nominal sample width (one extra bit for a side channel)
            if (d.channel_assignment == 9) bits += (c == 0);
            else if (d.channel_assignment == 8 || d.channel_assignment == 10) bits += (c == 1);
            // valid streams keep |sample| <= 2^(bits-1); anything beyond is caught by the check below
            narrow_ok = i32_acc_exact(absum, bits);
        }
    }
    PredRow pr;
    pr.out = active ? sub : nullptr;
    pr.bs = bs;
    pr.vec_ok = ((reinterpret_cast<uintptr_t>(sub) & 15) == 0) ? 1u : 0u;
    rows[lane] = pr;
    if (!__any_sync(0xffffffffu, active)) return;
    // idle lanes read (never write) the residuals of some active lane so that the bulk loop needs no guards
    const uint32_t some = __ffs(__ballot_sync(0xffffffffu, active)) - 1;
    const unsigned long long alias = __shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)sub, some);
    const int32_t* src = active ? sub : reinterpret_cast<const int32_t*>((uintptr_t)alias);
    __syncwarp();

    const uint32_t max_order = __reduce_max_sync(0xffffffffu, active ? order : 0u);
    const bool all_narrow = __all_sync(0xffffffffu, !active || narrow_ok);
    int32_t smin = 0, smax = 0;
    if (all_narrow) {
        if (max_order <= 4) predict_rows<4, 4, int>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        else if (max_order <= 8) predict_rows<8, 8, int>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        else if (max_order <= 12) predict_rows<12, 4, int>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        else predict_rows<32, 4, int>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        // exactness of the i32 accumulator: sum|coef| * max|sample| < 2^31 over the samples produced
        const uint32_t m = max((uint32_t)smax, 0u - (uint32_t)smin);
        if (active && order > 0 && (unsigned long long)absum * m >= (1ull << 31)) {
            results[f].status = CLX_INTERNAL_NEED_GENERIC;  // benign race: every writer stores the same value
            *need_generic = 1;
        }
    } else {
        if (max_order <= 4) predict_rows<4, 4, long long>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        else if (max_order <= 8) predict_rows<8, 8, long long>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        else if (max_order <= 12) predict_rows<12, 4, long long>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
        else predict_rows<32, 4, long long>(src, bs, order, shift, wasted, ca, second, coefs, active, tile, rows, s_ring[warp] + lane * RING_LANE_WORDS, lane, smin, smax);
    }
}

// ---------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------
size_t coop_params_bytes(const Plan& plan, uint32_t n_frames) {
    switch (plan.path) {
        case Path::LanePerFrame: return seq_scratch_bytes(plan, n_frames);
        case Path::WarpPerFrame: return (size_t)n_frames * plan.channels * sizeof(SubParams);
        case Path::Generic: break;
    }
    return 0;
}

cudaError_t launch_warp_per_frame(const uint8_t* d_bytes, uint64_t buf_bytes, const clx_frame_desc* d_descs, uint32_t n_frames,
                                  int32_t* d_out, clx_frame_result* d_results, int* d_need_generic, void* d_params,
                                  const Plan& plan, cudaStream_t stream, uint64_t* launches) {
    SubParams* params = reinterpret_cast<SubParams*>(d_params);
    const uint32_t CH = plan.channels;
    dim3 g1((n_frames + ENT_WARPS - 1) / ENT_WARPS), b1(ENT_WARPS * 32);
    entropy_frames_kernel<<<g1, b1, 0, stream>>>(d_bytes, buf_bytes, d_descs, n_frames, d_out, d_results, params, CH,
                                                 d_need_generic);
    (*launches)++;
    const uint64_t slots = (uint64_t)n_frames * CH;
    dim3 g2((uint32_t)((slots + PRE_WARPS * 32 - 1) / (PRE_WARPS * 32))), b2(PRE_WARPS * 32);
    predict_frames_kernel<<<g2, b2, 0, stream>>>(d_descs, n_frames, d_out, d_results, params, CH, d_need_generic);
    (*launches)++;
    return cudaGetLastError();
}

}  // namespace clx
