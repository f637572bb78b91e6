// Inner-loop shoot-out for one resampling pass over shared memory (H100):
//   A: current scheme  -- LDS.32 = 1 tap of 4 lines, PRMT + IMAD per tap and line (7 taps)
//   B: dp4a scheme     -- per output byte: 3 LDS.32, 2 funnel shifts, 6 IDP.4A (8 taps, 3 coefficient planes)
// Both produce u8 outputs into shared memory; bytes/clk/SM reported.  256 thr x 4 CTAs/SM.
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>
#define ITERS 64
__device__ __forceinline__ uint32_t fin(int a) { return (uint32_t)__vimin_s32_relu(a >> 22, 255); }

__global__ void __launch_bounds__(256, 4) kA(int* out, const int* coef) {
    __shared__ uint32_t in[32 * 160];     // planar row-packed words
    __shared__ uint8_t mid[44 * 388];
    for (int i = threadIdx.x; i < 32 * 160; i += 256) in[i] = i * 2654435761u;
    int k[7];
    for (int t = 0; t < 7; ++t) k[t] = coef[(threadIdx.x % 128) * 8 + 1 + t];
    const int first = coef[(threadIdx.x % 128) * 8] & 15;
    __syncthreads();
    const int px = threadIdx.x % 128, sub = threadIdx.x / 128;
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll 2
        for (int u = sub; u < 30; u += 2) {
            const uint32_t* wp = in + u * 160 + first + (px >> 3);
            uint32_t w[7];
#pragma unroll
            for (int t = 0; t < 7; ++t) w[t] = wp[t];
            int acc[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
#pragma unroll
            for (int t = 0; t < 7; ++t)
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[r] += (int)__byte_perm(w[t], 0, 0x4440 + r) * k[t];
            const int g = u / 3, c = u - g * 3;
            uint8_t* o = mid + (4 * g) * 388 + px * 3 + c;
#pragma unroll
            for (int r = 0; r < 4; ++r) o[r * 388] = (uint8_t)fin(acc[r]);
        }
        __syncthreads();
    }
    out[blockIdx.x * 256 + threadIdx.x] = mid[threadIdx.x];
}

__device__ __forceinline__ int dpu(uint32_t a, uint32_t b, int c) { int d; asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dps(uint32_t a, uint32_t b, int c) { int d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }

__global__ void __launch_bounds__(256, 4) kB(int* out, const int* coef) {
    __shared__ uint32_t inP[3 * 40 * 40];   // planar bytes: [c][row][160 bytes]
    __shared__ uint8_t midT[384 * 44];
    for (int i = threadIdx.x; i < 3 * 40 * 40; i += 256) inP[i] = i * 2654435761u;
    uint32_t K[6];
    for (int t = 0; t < 6; ++t) K[t] = coef[(threadIdx.x % 128) * 8 + 1 + t];
    const int first = coef[(threadIdx.x % 128) * 8] & 15;
    __syncthreads();
    const int px = threadIdx.x % 128, sub = threadIdx.x / 128;
    const int pos = first + px;            // byte position in the planar row
    const int sh = 8 * (pos & 3);
    const uint32_t* base = inP + (pos >> 2);
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll 4
        for (int u = sub; u < 120; u += 2) {     // (row, channel) pairs: 40 rows x 3
            const uint32_t* wp = base + u * 40;
            const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2];
            const uint32_t a = __funnelshift_r(w0, w1, sh), b = __funnelshift_r(w1, w2, sh);
            int a0 = dpu(a, K[0], 1 << 21); a0 = dpu(b, K[1], a0);
            int a1 = dpu(a, K[2], 0); a1 = dpu(b, K[3], a1);
            int a2 = dps(a, K[4], 0); a2 = dps(b, K[5], a2);
            const int acc = a0 + (a1 << 8) + (a2 << 16);
            const int row = u / 3, c = u - row * 3;
            midT[(px * 3 + c) * 44 + row] = (uint8_t)fin(acc);
        }
        __syncthreads();
    }
    out[blockIdx.x * 256 + threadIdx.x] = midT[threadIdx.x];
}

template <class F> void run(const char* name, F f, double bytes_per_iter) {
    int *out, *coef; cudaMalloc(&out, 132 * 4 * 256 * 4); cudaMalloc(&coef, 128 * 8 * 4); cudaMemset(coef, 1, 128 * 8 * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    f<<<132 * 4, 256>>>(out, coef);
    cudaEventRecord(e0); f<<<132 * 4, 256>>>(out, coef); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("%-10s %8.3f ms  %.2f output bytes/clk/SM  (%s)\n", name, ms, bytes_per_iter * ITERS * 4 / (ms * 1e-3 * 1.98e9), cudaGetErrorString(cudaGetLastError()));
}
int main() {
    run("A prmt+imad", kA, 30.0 * 4 * 128);     // per CTA per iter: 30 units x 4 rows x 128 px bytes
    run("B dp4a", kB, 120.0 * 128);
    return 0;
}
