// Pipe-throughput microbenchmark (H100): which integer/fp MAC form is fastest per SM?
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipes pipes.cu && ./pipes
#include <cstdio>
#include <cuda_runtime.h>
#define ITERS 4096
template <int MODE>
__global__ void k(int* out, int a0, int b0, float fa, float fb) {
    int acc[8]; float facc[8];
    int x[8]; float fx[8];
    for (int i = 0; i < 8; ++i) { acc[i] = threadIdx.x + i; x[i] = a0 + i * 3 + threadIdx.x; facc[i] = fa * i; fx[i] = fb + i + threadIdx.x; }
    int kk = b0; float fk = fb;
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (MODE == 0) acc[i] = x[i] * kk + acc[i];                       // IMAD r,r,r
            if (MODE == 1) facc[i] = fmaf(fx[i], fk, facc[i]);               // FFMA r,r,r
            if (MODE == 2) acc[i] = __dp4a(x[i], kk, acc[i]);                // IDP4A
            if (MODE == 3) acc[i] = __byte_perm(acc[i], x[i], 0x4140 + (it & 1)); // PRMT
            if (MODE == 4) { acc[i] = x[i] * kk + acc[i]; x[i] = __byte_perm(x[i], acc[(i+1)&7], 0x4321); }  // IMAD + PRMT pair
            if (MODE == 5) acc[i] = x[i] * 12345 + acc[i];                    // IMAD imm
            if (MODE == 6) { acc[i] = x[i] * kk + acc[i]; facc[i] = fmaf(fx[i], fk, facc[i]); } // IMAD + FFMA mix
            if (MODE == 7) acc[i] = (acc[i] >> 3) + x[i];                    // SHF+IADD (alu)
            if (MODE == 8) acc[i] = __vadd2(acc[i], x[i]);                    // packed add
            if (MODE == 9) acc[i] = min(max(acc[i] + x[i], 0), 255);         // add+clamp
        }
        kk += (MODE == 5) ? 0 : 1;
    }
    int s = 0; float fs = 0;
    for (int i = 0; i < 8; ++i) { s += acc[i]; fs += facc[i]; }
    out[blockIdx.x * blockDim.x + threadIdx.x] = s + (int)fs;
}
template <int MODE> void run(const char* name, int ops_per_iter) {
    int* out; cudaMalloc(&out, 132 * 8 * 1024 * sizeof(int));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<MODE><<<132 * 8, 256>>>(out, 1, 2, 1.f, 2.f);
    cudaEventRecord(e0);
    k<MODE><<<132 * 8, 256>>>(out, 1, 2, 1.f, 2.f);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double n = 132.0 * 8 * 256 * ITERS * 8 * ops_per_iter;
    printf("%-28s %8.3f ms  %8.2f Tlane-op/s  (%.1f lane-ops/clk/SM @1.98GHz)\n", name, ms, n / ms / 1e9, n / (ms * 1e-3) / 132 / 1.98e9);
    cudaFree(out);
}
int main() {
    run<0>("IMAD r,r,r", 1); run<5>("IMAD r,imm,r", 1); run<1>("FFMA r,r,r", 1); run<2>("IDP4A", 1); run<3>("PRMT", 1);
    run<4>("IMAD+PRMT (2 ops)", 2); run<6>("IMAD+FFMA (2 ops)", 2); run<7>("SHF+IADD (2 ops)", 2); run<8>("VADD2", 1); run<9>("IADD+MNMX x2 (3 ops)", 3);
    return 0;
}
