// pipebench.cu — issue-rate microbenchmark of the sm_90a pipes the 254-bit field arithmetic can use.
// Prints warp-instructions per clock per SM for IMAD.WIDE.U32, IMAD, IMAD.HI, DFMA, IADD3 and mixes.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipebench tools/pipebench.cu ; run on the GPU box.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITERS 2048
template <int MODE>
__global__ void __launch_bounds__(1024) k(uint64_t* out, uint32_t a, uint32_t b, double da, double db) {
    uint64_t x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
    uint32_t y0 = threadIdx.x, y1 = y0 + 1, y2 = y0 + 2, y3 = y0 + 3, y4 = y0 + 4, y5 = y0 + 5, y6 = y0 + 6, y7 = y0 + 7;
    double d0 = threadIdx.x, d1 = d0 + 1, d2 = d0 + 2, d3 = d0 + 3, d4 = d0 + 4, d5 = d0 + 5, d6 = d0 + 6, d7 = d0 + 7;
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < ITERS; i++) {
#define WIDE(x, m) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(x) : "r"((uint32_t)(m)), "r"(b))
#define LO(y, m) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(y) : "r"(m), "r"(b))
#define HI(y, m) asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(y) : "r"(m), "r"(b))
#define DF(d, m) asm volatile("fma.rn.f64 %0, %1, %2, %0;" : "+d"(d) : "d"(m), "d"(db))
#define AD(y, m) asm volatile("add.u32 %0, %0, %1;" : "+r"(y) : "r"(m))
#define ALL8(M, p) M(p##0, p##1); M(p##1, p##2); M(p##2, p##3); M(p##3, p##4); M(p##4, p##5); M(p##5, p##6); M(p##6, p##7); M(p##7, p##0)
        if (MODE == 0) { ALL8(WIDE, x); ALL8(WIDE, x); }
        if (MODE == 1) { ALL8(LO, y); ALL8(LO, y); }
        if (MODE == 2) { ALL8(HI, y); ALL8(HI, y); }
        if (MODE == 3) { ALL8(DF, d); ALL8(DF, d); }
        if (MODE == 4) { ALL8(AD, y); ALL8(AD, y); }
        if (MODE == 5) { ALL8(WIDE, x); ALL8(DF, d); }   // mix: do the pipes overlap?
        if (MODE == 6) { ALL8(LO, y); ALL8(DF, d); }
        if (MODE == 7) { ALL8(WIDE, x); ALL8(AD, y); }
    }
    long long t1 = clock64();
    uint64_t s = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7 + y0 + y1 + y2 + y3 + y4 + y5 + y6 + y7 +
                 (uint64_t)(d0 + d1 + d2 + d3 + d4 + d5 + d6 + d7);
    if (s == 0x1234567) out[0] = s;
    if (threadIdx.x == 0) out[1 + blockIdx.x] = (uint64_t)(t1 - t0);
}

template <int MODE>
void run(const char* name, uint64_t* d_out, int blocks) {
    k<MODE><<<blocks, 1024>>>(d_out, 12345u, 67891u, 1.0000001, 0.9999999);
    cudaDeviceSynchronize();
    uint64_t h[2];
    cudaMemcpy(h, d_out, 16, cudaMemcpyDeviceToHost);
    double cycles = (double)h[1];
    double winstr = 16.0 * ITERS * 32;  // warp-instructions per SM (32 warps)
    printf("%-28s %8.0f cycles  %6.3f warp-instr/clk/SM  (%5.1f lanes/clk/SM)\n", name, cycles, winstr / cycles, 32 * winstr / cycles);
}

int main() {
    uint64_t* d_out;
    cudaMalloc(&d_out, 8 * 4096);
    int sms = 132;
    run<0>("IMAD.WIDE.U32", d_out, sms);
    run<1>("IMAD (lo)", d_out, sms);
    run<2>("IMAD.HI.U32", d_out, sms);
    run<3>("DFMA", d_out, sms);
    run<4>("IADD", d_out, sms);
    run<5>("IMAD.WIDE + DFMA (1:1)", d_out, sms);
    run<6>("IMAD lo + DFMA (1:1)", d_out, sms);
    run<7>("IMAD.WIDE + IADD (1:1)", d_out, sms);
    return 0;
}
