// Which pipe does IDP.4A share?  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipes2 pipes2.cu
#include <cstdio>
#include <cuda_runtime.h>
#define ITERS 4096
template <int MODE>
__global__ void k(int* out, int a0, int b0) {
    int acc[8], x[8], y[8];
    for (int i = 0; i < 8; ++i) { acc[i] = threadIdx.x + i; x[i] = a0 + i * 3 + threadIdx.x; y[i] = x[i] * 7; }
    int kk = b0;
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (MODE == 0) { acc[i] = __dp4a(x[i], kk, acc[i]); y[i] = __funnelshift_r(y[i], acc[(i + 1) & 7], kk & 24); }   // IDP + SHF
            if (MODE == 1) { acc[i] = __dp4a(x[i], kk, acc[i]); y[i] = y[i] * kk + x[i]; }                                // IDP + IMAD
            if (MODE == 2) { acc[i] = __dp4a(x[i], kk, acc[i]); y[i] = __byte_perm(y[i], acc[(i + 1) & 7], 0x4321); }     // IDP + PRMT
            if (MODE == 3) { acc[i] = __dp4a((unsigned)x[i], (unsigned)kk, (unsigned)acc[i]); }                           // IDP u8.u8
            if (MODE == 4) { y[i] = __funnelshift_r(y[i], x[i], kk & 24); acc[i] = __byte_perm(acc[i], y[i], 0x4321); }     // SHF + PRMT (both ALU?)
            if (MODE == 5) { y[i] = __vimin_s32_relu(y[i] + x[i], 255); }                                                  // VIADD + VIMNMX.RELU
        }
        kk += 1;
    }
    int s = 0;
    for (int i = 0; i < 8; ++i) s += acc[i] + y[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int MODE> void run(const char* name, int ops) {
    int* out; cudaMalloc(&out, 132 * 8 * 256 * sizeof(int));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<MODE><<<132 * 8, 256>>>(out, 1, 2);
    cudaEventRecord(e0);
    k<MODE><<<132 * 8, 256>>>(out, 1, 2);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double n = 132.0 * 8 * 256 * ITERS * 8 * ops;
    printf("%-28s %8.3f ms  %.1f lane-ops/clk/SM\n", name, ms, n / (ms * 1e-3) / 132 / 1.98e9);
    cudaFree(out);
}
int main() {
    run<0>("IDP4A + SHF", 2); run<1>("IDP4A + IMAD", 2); run<2>("IDP4A + PRMT", 2); run<3>("IDP4A u8.u8", 1);
    run<4>("SHF + PRMT", 2); run<5>("VIADD + VIMNMX.RELU", 2);
    return 0;
}
