// ubench_pipes.cu — issue-rate microbenchmarks for the integer instructions the decode kernels lean on.
// Each kernel runs 8 independent dependency chains per thread of one instruction kind; with 16 warps per SM
// sub-partition the result is the pipe's throughput in warp-instructions per cycle per sub-partition.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/scratch/ubench_pipes tools/ubench_pipes.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define ITERS 2048
#define CHAINS 8

#define KERNEL(name, ASM)                                                                             \
    __global__ void name(uint32_t* out, uint32_t seed, long long* cyc) {                              \
        uint32_t r[CHAINS];                                                                           \
        for (int i = 0; i < CHAINS; i++) r[i] = seed + threadIdx.x * 31 + i * 7;                      \
        uint32_t b = seed | 5u, c = (seed >> 3) | 9u;                                                 \
        __syncthreads();                                                                              \
        long long t0 = clock64();                                                                     \
        for (int it = 0; it < ITERS; it++) {                                                          \
            _Pragma("unroll") for (int i = 0; i < CHAINS; i++) { ASM; }                               \
        }                                                                                             \
        long long t1 = clock64();                                                                     \
        uint32_t s = 0;                                                                               \
        for (int i = 0; i < CHAINS; i++) s ^= r[i];                                                   \
        out[blockIdx.x * blockDim.x + threadIdx.x] = s;                                               \
        if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;                                              \
    }

KERNEL(k_iadd3, asm volatile("add.u32 %0, %0, %1;" : "+r"(r[i]) : "r"(b)))
KERNEL(k_lop3, asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(r[i]) : "r"(b), "r"(c)))
KERNEL(k_shf_wrap, asm volatile("shf.l.wrap.b32 %0, %0, %1, %2;" : "+r"(r[i]) : "r"(b), "r"(c)))
KERNEL(k_shr, asm volatile("shf.r.clamp.b32 %0, %0, %1, %2;" : "+r"(r[i]) : "r"(c), "r"(b & 3u)))
KERNEL(k_prmt, asm volatile("prmt.b32 %0, %0, %1, 0x0123;" : "+r"(r[i]) : "r"(b)))
KERNEL(k_sgxt, asm volatile("bfe.s32 %0, %0, 0, 17;" : "+r"(r[i])))
KERNEL(k_imad, asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(r[i]) : "r"(b), "r"(c)))
KERNEL(k_flo, asm volatile("bfind.u32 %0, %0; or.b32 %0, %0, %1;" : "+r"(r[i]) : "r"(b)))
KERNEL(k_popc, asm volatile("popc.b32 %0, %0; or.b32 %0, %0, %1;" : "+r"(r[i]) : "r"(b)))
KERNEL(k_vimnmx, asm volatile("max.u32 %0, %0, %1;" : "+r"(r[i]) : "r"(b)))
KERNEL(k_setp_sel, asm volatile("{ .reg .pred p; setp.lt.u32 p, %0, %1; selp.u32 %0, %2, %0, p; }" : "+r"(r[i]) : "r"(b), "r"(c)))


// 64-bit chains: the i64 accumulate of the prediction (IMAD.WIDE) against its double-precision equivalent
// (DFMA is exact for these products: 15-bit coefficients x 25-bit samples, sums below 2^53) and the conversions
// the latter would need once per sample.
#define KERNEL64(name, T, INIT, ASM)                                                                  \
    __global__ void name(uint32_t* out, uint32_t seed, long long* cyc) {                              \
        T r[CHAINS];                                                                                  \
        for (int i = 0; i < CHAINS; i++) r[i] = (T)(INIT);                                            \
        int b = (int)(seed | 5u), c = (int)((seed >> 3) | 9u);                                        \
        double db = (double)b, dc = 1.0 / (double)c;                                                  \
        __syncthreads();                                                                              \
        long long t0 = clock64();                                                                     \
        for (int it = 0; it < ITERS; it++) {                                                          \
            _Pragma("unroll") for (int i = 0; i < CHAINS; i++) { ASM; }                               \
        }                                                                                             \
        long long t1 = clock64();                                                                     \
        T s = 0;                                                                                      \
        for (int i = 0; i < CHAINS; i++) s += r[i];                                                   \
        out[blockIdx.x * blockDim.x + threadIdx.x] = (uint32_t)(long long)s + (uint32_t)(db + dc);    \
        if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;                                              \
    }
KERNEL64(k_imad_wide, long long, seed + threadIdx.x * 31 + i * 7, asm volatile("mad.wide.s32 %0, %1, %2, %0;" : "+l"(r[i]) : "r"((int)r[i]), "r"(c)))
KERNEL64(k_dfma, double, seed + threadIdx.x * 31 + i * 7, asm volatile("fma.rn.f64 %0, %1, %2, %0;" : "+d"(r[i]) : "d"(db), "d"(dc)))
KERNEL64(k_cvt_rt, double, seed + threadIdx.x * 31 + i * 7,
         { long long q; asm volatile("cvt.rzi.s64.f64 %0, %1;" : "=l"(q) : "d"(r[i])); int lo = (int)(q >> 3) + b; asm volatile("cvt.rn.f64.s32 %0, %1;" : "=d"(r[i]) : "r"(lo)); })

__global__ void k_lds(uint32_t* out, uint32_t seed, long long* cyc) {  // dependent shared-memory loads, conflict-free
    __shared__ uint32_t s[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = (i + 32) & 1023;
    __syncthreads();
    uint32_t idx[CHAINS];
    for (int i = 0; i < CHAINS; i++) idx[i] = (threadIdx.x + 32 * i) & 1023;
    long long t0 = clock64();
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < CHAINS; i++) idx[i] = s[idx[i]];
    }
    long long t1 = clock64();
    uint32_t x = 0;
    for (int i = 0; i < CHAINS; i++) x ^= idx[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = x + seed;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <typename K>
void run(const char* name, K kern, int threads, double ops_per_chain_step) {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    uint32_t* out;
    long long* cyc;
    cudaMalloc(&out, sizeof(uint32_t) * sms * threads);
    cudaMalloc(&cyc, sizeof(long long) * sms);
    kern<<<sms, threads>>>(out, 12345u, cyc);
    kern<<<sms, threads>>>(out, 12345u, cyc);
    cudaDeviceSynchronize();
    long long h[1024];
    cudaMemcpy(h, cyc, sizeof(long long) * sms, cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < sms; i++) avg += (double)h[i];
    avg /= sms;
    const double warp_insts = (double)ITERS * CHAINS * ops_per_chain_step * (threads / 32);
    printf("%-24s threads/SM %4d: %8.0f cycles, %.3f warp-inst/clk/SM (%.3f per sub-partition), dependent-op latency ~%.1f clk at 1 warp\n", name,
           threads, avg, warp_insts / avg, warp_insts / avg / 4, avg / ((double)ITERS * ops_per_chain_step) );
    cudaFree(out);
    cudaFree(cyc);
}

int main() {
    for (int threads : {32, 512, 1024}) {
        printf("---- %d threads per SM (%d warps per sub-partition)\n", threads, threads / 128 ? threads / 128 : 1);
        run("IADD3 (2 adds fused)", k_iadd3, threads, 0.5);
        run("LOP3", k_lop3, threads, 1);
        run("SHF.W", k_shf_wrap, threads, 1);
        run("SHF.R.clamp", k_shr, threads, 1);
        run("PRMT", k_prmt, threads, 1);
        run("SGXT(bfe)", k_sgxt, threads, 1);
        run("IMAD", k_imad, threads, 1);
        run("FLO+LOP", k_flo, threads, 2);
        run("POPC+LOP", k_popc, threads, 2);
        run("VIMNMX3 (2 max fused)", k_vimnmx, threads, 0.5);
        run("SETP+SEL", k_setp_sel, threads, 2);
        run("LDS chain", k_lds, threads, 1);
        run("IMAD.WIDE (s32xs32+s64)", k_imad_wide, threads, 1);
        run("DFMA", k_dfma, threads, 1);
        run("F2I.S64.F64 + I2F.F64.S32 (+shift,add)", k_cvt_rt, threads, 2);
    }
    return 0;
}
