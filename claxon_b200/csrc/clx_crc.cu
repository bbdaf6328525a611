// clx_crc.cu — the frame CRC-16 check (reference src/frame.rs:752-763, src/crc.rs:60-112: polynomial 0x8005,
// initial value 0, bits MSB first, no reflection, no final xor) on the device, one WARP per frame.
//
// The frame's bytes [0, n) (sync code up to, not including, the two footer bytes) are right-aligned in a virtual
// message of 32 * C bytes, C a power of two: leading zero bytes do not change a CRC whose initial value is 0.  Lane l
// takes the virtual bytes [l * C, (l + 1) * C) with a table-driven CRC (four 256-entry tables, a word per step), and
// the 32 partial values are combined pairwise over five levels: crc(A || B) = crc(A) * x^(8 |B|) + crc(B) in
// GF(2)[x] / P(x), the factors x^(8 * 2^j) mod P coming from a table built once on the host.  n = the length the
// decode kernels found (`consumed` - 2), so a frame whose boundary was only a guess is checked over what it really
// spans.  A mismatch turns CLX_OK into CLX_ERR_FRAME_CRC_MISMATCH; a frame that failed to decode keeps its error
// (the reference reports subframe errors first, the CRC only after all subframes decoded).
#include <cuda_runtime.h>
#include <stdint.h>

#include "claxon_b200.h"
#include "clx_internal.h"

namespace clx {

constexpr int CRC_WARPS = 8;

struct CrcPowers { uint16_t p[32]; };  // p[j] = x^(8 * 2^j) mod P

// a * b in GF(2)[x] / (x^16 + x^15 + x^2 + 1), both of degree < 16
__host__ __device__ inline uint32_t crc_mulmod(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int i = 15; i >= 0; i--) {
        r <<= 1;
        if (r & 0x10000u) r ^= 0x18005u;
        if ((b >> i) & 1u) r ^= a;
    }
    return r;
}

static CrcPowers host_powers() {
    CrcPowers t;
    uint32_t v = 0x0100;  // x^8
    for (int j = 0; j < 32; j++) { t.p[j] = (uint16_t)v; v = crc_mulmod(v, v); }
    return t;
}

// Slicing-by-4 tables, built once on the host: t[k][b] = CRC of byte b followed by k zero bytes.
struct CrcTables { uint16_t t[4][256]; };
__device__ CrcTables g_crc_tables;

static CrcTables host_tables() {
    CrcTables T;
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t d = i << 8;
        for (int k = 0; k < 8; k++) d = (d & 0x8000u) ? ((d << 1) ^ 0x8005u) & 0xffffu : (d << 1) & 0xffffu;
        T.t[0][i] = (uint16_t)d;
    }
    for (int k = 1; k < 4; k++)
        for (uint32_t i = 0; i < 256; i++) {
            const uint32_t v = T.t[k - 1][i];
            T.t[k][i] = (uint16_t)(((v << 8) & 0xffffu) ^ T.t[0][v >> 8]);
        }
    return T;
}

__global__ void __launch_bounds__(CRC_WARPS * 32)
crc16_frames_kernel(const uint8_t* __restrict__ bytes, const clx_frame_desc* __restrict__ descs, uint32_t n_frames,
                    clx_frame_result* __restrict__ results, CrcPowers pw) {
    __shared__ uint16_t s_t[4][256];
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&g_crc_tables);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&s_t[0][0]);
        for (uint32_t i = threadIdx.x; i < 512; i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t f = blockIdx.x * CRC_WARPS + (threadIdx.x >> 5);
    if (f >= n_frames) return;
    const clx_frame_result res = results[f];
    if (res.status != CLX_OK) return;
    const clx_frame_desc d = descs[f];
    if ((d.flags & CLX_FRAME_CRC16_VERIFIED) && res.consumed == d.byte_len) return;  // the demuxer matched it already
    if (res.consumed < 2 || res.consumed > d.byte_len) {  // cannot happen for a frame that decoded; be safe
        if (lane == 0) results[f].status = CLX_ERR_FRAME_CRC_MISMATCH;
        return;
    }
    const uint32_t n = res.consumed - 2;
    const uint8_t* p = bytes + d.byte_offset;
    uint32_t s = 0;  // log2 of the chunk size
    while ((32u << s) < n) s++;
    const uint32_t C = 1u << s, pad = 32u * C - n;
    // this lane's virtual bytes [lo, hi) -> real bytes [lo - pad, hi - pad)
    const uint32_t vlo = lane * C, vhi = vlo + C;
    uint32_t a = vlo > pad ? vlo - pad : 0u, b = vhi > pad ? vhi - pad : 0u;
    uint32_t crc = 0;
    auto byte_step = [&](uint32_t x) { crc = ((crc << 8) & 0xffffu) ^ s_t[0][(crc >> 8) ^ x]; };
    // little-endian word: first byte in bits 0-7.  Only two of the four lookups depend on the running value.
    auto word_step = [&](uint32_t w) {
        crc = s_t[3][((crc >> 8) ^ w) & 0xffu] ^ s_t[2][((crc ^ (w >> 8)) & 0xffu)] ^ s_t[1][(w >> 16) & 0xffu] ^ s_t[0][w >> 24];
    };
    // head up to a 16-byte aligned address; 16-byte vectors, each loaded one iteration before it is used (the
    // addresses do not depend on the running value, so the loads overlap the table chain); tail
    while (a < b && ((uintptr_t)(p + a) & 15u)) { byte_step(p[a]); a++; }
    if (a + 16 <= b) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(p + a));
        for (; a + 32 <= b; a += 16) {
            const uint4 nx = __ldg(reinterpret_cast<const uint4*>(p + a + 16));
            word_step(v.x); word_step(v.y); word_step(v.z); word_step(v.w);
            v = nx;
        }
        word_step(v.x); word_step(v.y); word_step(v.z); word_step(v.w);
        a += 16;
    }
    while (a < b) { byte_step(p[a]); a++; }
    // combine: after level j a lane holds the CRC of 2^(j+1) chunks (valid in lanes whose low j+1 bits are all ones)
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const uint32_t left = __shfl_up_sync(0xffffffffu, crc, 1u << j);   // the run of chunks just before this one
        if ((lane & ((2u << j) - 1u)) == (2u << j) - 1u) crc = crc_mulmod(left, pw.p[s + j]) ^ crc;
    }
    if (lane == 31) {
        const uint32_t stored = ((uint32_t)p[n] << 8) | p[n + 1];
        if (crc != stored) results[f].status = CLX_ERR_FRAME_CRC_MISMATCH;
    }
}

// Uploads the tables to the CURRENT device (a __device__ symbol has one instance per device); called once per
// context from clx_ctx_create, never from inside a stream capture.
cudaError_t crc16_init() {
    static const CrcTables T = host_tables();
    return cudaMemcpyToSymbol(g_crc_tables, &T, sizeof T);
}

cudaError_t launch_crc16(const uint8_t* d_bytes, const clx_frame_desc* d_descs, uint32_t n_frames, clx_frame_result* d_results,
                         cudaStream_t stream, uint64_t* launches) {
    if (n_frames == 0) return cudaSuccess;
    static const CrcPowers pw = host_powers();
    crc16_frames_kernel<<<(n_frames + CRC_WARPS - 1) / CRC_WARPS, CRC_WARPS * 32, 0, stream>>>(d_bytes, d_descs, n_frames, d_results, pw);
    (*launches)++;
    return cudaGetLastError();
}

}  // namespace clx
