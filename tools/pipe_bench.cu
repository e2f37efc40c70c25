// Development aid: issue throughput of the integer instructions K1 is made of (per SM sub-partition).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipe_bench tools/pipe_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITER 2048
template <int OP>
__global__ void k(uint32_t* out, uint32_t seed, unsigned long long* cyc) {
    uint32_t a[8];
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = seed * (threadIdx.x + 1) + i * 0x9e3779b9u;
    unsigned long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < ITER; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint32_t x = a[i], y = a[(i + 1) & 7];
            if (OP == 0) asm volatile("lop3.b32 %0, %0, %1, 0x0f0f0f0f, 0xE4;" : "+r"(x) : "r"(y));
            if (OP == 1) asm volatile("shr.u32 %0, %0, 4; xor.b32 %0, %0, %1;" : "+r"(x) : "r"(y));  // SHF + LOP3
            if (OP == 2) asm volatile("mul.hi.u32 %0, %0, 0x10000000; xor.b32 %0, %0, %1;" : "+r"(x) : "r"(y));  // IMAD.HI + LOP3
            if (OP == 3) asm volatile("shl.b32 %0, %0, 4; xor.b32 %0, %0, %1;" : "+r"(x) : "r"(y));  // IMAD.SHL/SHF + LOP3
            if (OP == 4) asm volatile("mul.hi.u32 %0, %0, 0x10000001;" : "+r"(x));                  // IMAD.HI alone
            if (OP == 5) asm volatile("mad.lo.u32 %0, %0, 0x11, %1;" : "+r"(x) : "r"(y));            // IMAD alone
            if (OP == 6) asm volatile("prmt.b32 %0, %0, %1, 0x5140;" : "+r"(x) : "r"(y));
            if (OP == 7) asm volatile("bfind.u32 %0, %0; add.u32 %0, %0, %1;" : "+r"(x) : "r"(y));   // FLO + IADD
            if (OP == 8) asm volatile("mad.lo.u32 %0, %0, 0x11, %1; xor.b32 %0, %0, %1;" : "+r"(x) : "r"(y));  // IMAD + LOP3
            if (OP == 9) asm volatile("shf.l.wrap.b32 %0, %0, %1, 7;" : "+r"(x) : "r"(y));
            a[i] = x;
        }
    }
    unsigned long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s ^= a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int OP>
void run(const char* name, int ninstr) {
    uint32_t* out;
    unsigned long long* cyc;
    const int threads = 512, blocks = 148;  // 16 warps per SM = 4 per sub-partition
    cudaMalloc(&out, blocks * threads * 4);
    cudaMalloc(&cyc, blocks * 8);
    k<OP><<<blocks, threads>>>(out, 12345, cyc);
    k<OP><<<blocks, threads>>>(out, 12345, cyc);
    cudaDeviceSynchronize();
    unsigned long long h[148];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    double c = 0;
    for (int i = 0; i < blocks; i++) c += h[i];
    c /= blocks;
    double warp_instr_per_smsp = (double)ITER * 8 * ninstr * 4;  // 4 warps per sub-partition
    printf("%-28s %6.3f warp-instr / cycle / sub-partition  (%d instr per op)\n", name, warp_instr_per_smsp / c, ninstr);
    cudaFree(out);
    cudaFree(cyc);
}

int main() {
    run<0>("LOP3", 1);
    run<9>("SHF", 1);
    run<6>("PRMT", 1);
    run<5>("IMAD", 1);
    run<4>("IMAD.HI", 1);
    run<1>("SHF.R + LOP3", 2);
    run<3>("SHL + LOP3", 2);
    run<2>("IMAD.HI + LOP3", 2);
    run<8>("IMAD + LOP3", 2);
    run<7>("FLO + IADD", 2);
    return 0;
}
