// ubench.cu — issue-rate microbenchmarks for the integer pipes on sm_90a
// (nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu).
//   which instruction mixes overlap?  IMAD.WIDE.U32(.X) vs IADD3(.X) vs LOP3 vs 32-bit IMAD
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define DEV __device__ __forceinline__
DEV void madw(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) { asm volatile("mad.lo.cc.u32 %0,%2,%3,%0;\n\tmadc.hi.cc.u32 %1,%2,%3,%1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b)); }
DEV void madcw(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) { asm volatile("madc.lo.cc.u32 %0,%2,%3,%0;\n\tmadc.hi.cc.u32 %1,%2,%3,%1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b)); }
DEV uint32_t addcc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t addccc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }

// MODE: 0 = wide MAD chains only (NW per iter), 1 = add chains only (NA per iter), 2 = both
template <int NW, int NA, int PLAIN>
__global__ void k(uint32_t *out, int iters) {
    uint32_t a = threadIdx.x * 2654435761u + 1, b = blockIdx.x * 40503u + 7;
    uint32_t w[16], x[16];
#pragma unroll
    for (int i = 0; i < 16; i++) { w[i] = a + i; x[i] = b + i; }
    for (int it = 0; it < iters; it++) {
        if (NW > 0) {
            if (PLAIN) {
#pragma unroll
                for (int i = 0; i < NW; i++) { uint64_t t = (uint64_t)a * (b + i) + (((uint64_t)w[2 * (i % 8) + 1] << 32) | w[2 * (i % 8)]); w[2 * (i % 8)] = (uint32_t)t; w[2 * (i % 8) + 1] = (uint32_t)(t >> 32); }
            } else {
#pragma unroll
                for (int c = 0; c < NW / 4; c++) {  // chains of 4 wide MADs with carry
                    madw(w[0 + (c & 1) * 8], w[1 + (c & 1) * 8], a, b + c);
                    madcw(w[2 + (c & 1) * 8], w[3 + (c & 1) * 8], a, b);
                    madcw(w[4 + (c & 1) * 8], w[5 + (c & 1) * 8], a, b);
                    madcw(w[6 + (c & 1) * 8], w[7 + (c & 1) * 8], a, b);
                }
            }
        }
        if (NA > 0) {
#pragma unroll
            for (int c = 0; c < NA / 8; c++) {  // chains of 8 adds with carry
                x[0 + (c & 1) * 8] = addcc(x[0 + (c & 1) * 8], b);
#pragma unroll
                for (int i = 1; i < 8; i++) x[i + (c & 1) * 8] = addccc(x[i + (c & 1) * 8], a);
            }
        }
        a ^= w[3]; b += x[5];
    }
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += w[i] ^ x[i];
    if (s == 0x12345) out[0] = s;
}

template <int NW, int NA, int PLAIN>
void run(const char *name, uint32_t *d, int sms) {
    const int iters = 2048, blocks = sms * 4, threads = 512;
    k<NW, NA, PLAIN><<<blocks, threads>>>(d, 16);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e30f;
    for (int r = 0; r < 3; r++) {
        cudaEventRecord(e0); k<NW, NA, PLAIN><<<blocks, threads>>>(d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    double warps_per_smsp = (double)blocks * threads / 32 / (sms * 4);
    double cyc = best * 1e-3 * clk * 1e3;  // at nominal max clock
    double per_iter = cyc / iters / warps_per_smsp;  // SMSP cycles per warp-iteration
    printf("%-28s NW=%2d NA=%2d : %.3f ms  %.1f cyc/warp-iter  -> %.2f cyc per instr (of %d)\n", name, NW, NA, best, per_iter, per_iter / (NW + NA), NW + NA);
}

// SHFL mixes: what a limb-per-lane layout pays.  NS shuffles per iteration (each moves one 32-bit limb between lanes),
// optionally beside NW wide MADs.
template <int NW, int NS>
__global__ void ks(uint32_t *out, int iters) {
    uint32_t a = threadIdx.x * 2654435761u + 1, b = blockIdx.x * 40503u + 7;
    uint32_t w[16], x[8];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = a + i;
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = b + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int c = 0; c < NW / 4; c++) {
            madw(w[0 + (c & 1) * 8], w[1 + (c & 1) * 8], a, b + c);
            madcw(w[2 + (c & 1) * 8], w[3 + (c & 1) * 8], a, b);
            madcw(w[4 + (c & 1) * 8], w[5 + (c & 1) * 8], a, b);
            madcw(w[6 + (c & 1) * 8], w[7 + (c & 1) * 8], a, b);
        }
#pragma unroll
        for (int i = 0; i < NS; i++) x[i & 7] = __shfl_xor_sync(0xffffffffu, x[i & 7] + (uint32_t)i, 1 + (i & 3));
        a ^= w[3]; b += x[5];
    }
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += w[i];
#pragma unroll
    for (int i = 0; i < 8; i++) s ^= x[i];
    if (s == 0x12345) out[0] = s;
}
template <int NW, int NS>
void runs(const char *name, uint32_t *d, int sms) {
    const int iters = 2048, blocks = sms * 4, threads = 512;
    ks<NW, NS><<<blocks, threads>>>(d, 16);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e30f;
    for (int r = 0; r < 3; r++) {
        cudaEventRecord(e0); ks<NW, NS><<<blocks, threads>>>(d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    double warps_per_smsp = (double)blocks * threads / 32 / (sms * 4);
    double per_iter = best * 1e-3 * clk * 1e3 / iters / warps_per_smsp;
    printf("%-28s NW=%2d NS=%2d : %.3f ms  %.1f cyc/warp-iter  (SHFL+its add: %.2f cyc each when NW=0)\n", name, NW, NS, best, per_iter, NS ? per_iter / NS : 0.0);
}

int main() {
    uint32_t *d; cudaMalloc(&d, 4096);
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount;
    printf("%s SMs=%d\n", p.name, sms);
    run<32, 0, 1>("wide plain", d, sms);
    run<32, 0, 0>("wide carry-chain", d, sms);
    run<0, 32, 0>("add carry-chain", d, sms);
    run<0, 64, 0>("add carry-chain", d, sms);
    run<32, 32, 0>("mix wide:add 1:1", d, sms);
    run<32, 64, 0>("mix wide:add 1:2", d, sms);
    run<16, 64, 0>("mix wide:add 1:4", d, sms);
    run<32, 64, 1>("mix plainwide:add 1:2", d, sms);
    runs<0, 16>("shfl only", d, sms);
    runs<0, 32>("shfl only", d, sms);
    runs<32, 0>("wide only (same harness)", d, sms);
    runs<32, 16>("wide + 16 shfl", d, sms);
    runs<32, 32>("wide + 32 shfl", d, sms);
    return 0;
}
