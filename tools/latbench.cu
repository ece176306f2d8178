// latbench.cu — latency/throughput of chained G1 point additions for one warp vs many warps.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --expt-relaxed-constexpr -o tools/latbench tools/latbench.cu ; run on the GPU box.
#include <cstdio>
#include "../halo2-lib_b200/csrc/quad.cuh"
using namespace h2b;
__global__ void k_chain(const Affine* pts, XYZZ* out, int iters, long long* cyc) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    Affine p = Affine::load(pts + (t & 1023));
    XYZZ acc = xyzz_dbl_affine(p);
    XYZZ q = XYZZ::from_affine(Affine::load(pts + ((t + 7) & 1023)));
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; i++) { xyzz_add(acc, q); }
    long long t1 = clock64();
    acc.store(out + t);
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_quadchain(const Affine* pts, XYZZ* out, int iters, long long* cyc) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int q = t >> 2;
    Affine p = Affine::load(pts + (q & 1023));
    XYZZ acc = xyzz_dbl_affine(p);
    XYZZ a2 = XYZZ::from_affine(Affine::load(pts + ((q + 7) & 1023)));
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; i++) { quad_add(acc, a2); }
    long long t1 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; i++) { quad_dbl(acc); }
    long long t2 = clock64();
    acc.store(out + t);
    if (threadIdx.x == 0 && blockIdx.x == 0) { cyc[0] = t1 - t0; cyc[1] = t2 - t1; }
}
__global__ void k_mulchain(const uint64_t* in, uint64_t* out, int iters, long long* cyc) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    Fq a = Fq::load(in + 4 * (t & 1023)), b = Fq::load(in + 4 * ((t + 3) & 1023));
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; i++) { a = a * b; }
    long long t1 = clock64();
    a.store(out + 4 * t);
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_gen(Affine* pts) {  // 1024 valid points: multiples of G
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    Affine g; g.x = Fq::one(); g.y = Fq::one() + Fq::one();
    XYZZ acc = XYZZ::from_affine(g);
    for (int i = 0; i < t + 1; i++) xyzz_madd(acc, g);
    xyzz_to_affine(acc).store(pts + t);
}
int main() {
    Affine* pts; XYZZ* out; long long* cyc; uint64_t* fo;
    cudaMalloc(&pts, 1024 * sizeof(Affine)); cudaMalloc(&out, 132 * 1024 * sizeof(XYZZ)); cudaMalloc(&cyc, 8); cudaMalloc(&fo, 132*1024*32);
    k_gen<<<8, 128>>>(pts); cudaDeviceSynchronize();
    int iters = 200;
    struct { int blocks, threads; const char* name; } cfg[] = {{1, 32, "1 warp"}, {1, 128, "1 CTA x 4 warps (1/SMSP)"}, {132, 128, "132 CTA x 4 warps"}, {132, 512, "132 x 16 warps (4/SMSP)"}, {132, 1024, "132 x 32 warps (8/SMSP)"}};
    {
        long long h2[2];
        cudaFree(cyc); cudaMalloc(&cyc, 16);
        k_quadchain<<<1, 32>>>(pts, out, iters, cyc); cudaDeviceSynchronize();
        cudaMemcpy(h2, cyc, 16, cudaMemcpyDeviceToHost);
        printf("quad_add chain  1 warp (8 quads)   %8.0f cycles/op    quad_dbl chain %8.0f cycles/op\n", (double)h2[0] / iters, (double)h2[1] / iters);
        k_quadchain<<<132, 128>>>(pts, out, iters, cyc); cudaDeviceSynchronize();
        cudaMemcpy(h2, cyc, 16, cudaMemcpyDeviceToHost);
        printf("quad_add chain  132 x 4 warps      %8.0f cycles/op    quad_dbl chain %8.0f cycles/op\n", (double)h2[0] / iters, (double)h2[1] / iters);
    }
    for (auto& c : cfg) {
        long long h;
        k_chain<<<c.blocks, c.threads>>>(pts, out, iters, cyc); cudaDeviceSynchronize();
        cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        printf("xyzz_add chain  %-28s %8.0f cycles/op  (%.0f cycles per mult-equivalent /14)\n", c.name, (double)h / iters, (double)h / iters / 14);
        k_mulchain<<<c.blocks, c.threads>>>((uint64_t*)pts, fo, iters * 10, cyc); cudaDeviceSynchronize();
        cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        printf("Fq mul chain    %-28s %8.0f cycles/mul\n", c.name, (double)h / (iters * 10));
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
