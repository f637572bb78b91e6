// Tensor-core formulation of one 8-bit LANCZOS pass (H100, sm_90a): probe + shoot-out.
//
// A resampling pass is a banded integer contraction: out[o] = (2^21 + sum_k in[k] * coef[o][k]) >> 22 with 23-bit
// signed coefficients.  mma.sync.m16n8k32 multiplies u8 pixels by 8-bit coefficient LIMBS with exact s32
// accumulation: coef = c2 * 65536 + c1 * 256 + c0 (c0, c1 unsigned bytes, c2 signed), three MMAs per tile, recombined
// with two shift-adds.  |limb sums| <= 32 * 255 * 255 < 2^21, the recombined value is Pillow's accumulator exactly.
//
//   part 1  correctness of the fragment layout + mixed u8/s8 operand types against a scalar loop
//   part 2  raw IMMA issue rate (independent accumulators)
//   part 3  H pass:  M = 16 outputs (coefficient band matrix, registers), N = rows, K = 32 input pixels of a plane
//           V pass:  M = 16 output rows (coefficients, registers), N = byte columns, K = 32 input rows (row-packed)
//           reported as output bytes/clk/SM, to compare with taps.cu's "A prmt+imad"
//
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o imma imma.cu && ./imma
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#define ITERS 64

__device__ __forceinline__ void mma_uu(int (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2], const int (&c)[4]) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
                 : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]));
}
__device__ __forceinline__ void mma_su(int (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2], const int (&c)[4]) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
                 : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]));
}
__device__ __forceinline__ uint32_t fin(int a) { return (uint32_t)__vimin_s32_relu(a >> 22, 255); }

// ---- part 1: one warp, one 16 x 8 tile, K = 32 -------------------------------------------------------------------
// coefA: [3 limbs][16 m][32 k] bytes; in: [8 n][32 k] bytes; out: [16][8] int32 (the recombined accumulator)
__global__ void probe(const uint8_t* coefA, const uint8_t* in, int* out) {
    const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
    uint32_t a[3][4], b[2];
    for (int l = 0; l < 3; ++l) {
        const uint8_t* A = coefA + l * 512;
        a[l][0] = *(const uint32_t*)(A + g * 32 + 4 * t);
        a[l][1] = *(const uint32_t*)(A + (g + 8) * 32 + 4 * t);
        a[l][2] = *(const uint32_t*)(A + g * 32 + 16 + 4 * t);
        a[l][3] = *(const uint32_t*)(A + (g + 8) * 32 + 16 + 4 * t);
    }
    b[0] = *(const uint32_t*)(in + g * 32 + 4 * t);
    b[1] = *(const uint32_t*)(in + g * 32 + 16 + 4 * t);
    const int z[4] = {0, 0, 0, 0}, r[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
    int d0[4], d1[4], d2[4];
    mma_uu(d0, a[0], b, r);
    mma_uu(d1, a[1], b, z);
    mma_su(d2, a[2], b, z);
    for (int i = 0; i < 4; ++i) {
        const int row = g + (i >= 2 ? 8 : 0), col = 2 * t + (i & 1);
        out[row * 8 + col] = d0[i] + (d1[i] << 8) + (d2[i] << 16);
    }
}

// ---- part 2: raw issue rate ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 4) rate(int* out, int n_acc) {
    uint32_t a[4] = {threadIdx.x, threadIdx.x * 3u, threadIdx.x * 5u, 7u}, b[2] = {threadIdx.x * 11u, 13u};
    int acc[8][4];
    for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) acc[i][j] = i + j;
    for (int it = 0; it < ITERS * 16; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) mma_uu(acc[i], a, b, acc[i]);
    }
    int s = 0;
    for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) s += acc[i][j];
    out[blockIdx.x * 256 + threadIdx.x] = s;
}

// ---- part 3a: H pass ---------------------------------------------------------------------------------------------------
// planes: [3 channels][40 rows][PB bytes] u8, PB = 176 (rows 16-byte aligned; row skew keeps the 8 x 4 word reads of
// a fragment on distinct banks).  Warp w owns outputs 16w..16w+15 (a 128 px block).  mid: row-packed words
// word(kg, col) = rows 4kg..4kg+3 of byte column col = 3 * px + c, pitch 440 words (== 24 mod 32).
#define PB 176
#define MIDP 440
__device__ __forceinline__ int plane_off(int c, int row) { return (c * 40 + row) * PB + 32 * (row >> 3); }
__global__ void __launch_bounds__(256, 4) kH(int* out, const uint4* fragsA, const int* kx0s) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t* planes = sm;                                   // 3 * 40 * 176 + skew
    uint32_t* mid = (uint32_t*)(sm + 3 * 40 * PB + 32 * 5);   // 12 * 440 words (48 computed rows)
    for (int i = threadIdx.x; i < (3 * 40 * PB + 160) / 4; i += 256) ((uint32_t*)planes)[i] = i * 2654435761u;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    uint32_t a[3][4];
    for (int l = 0; l < 3; ++l) {
        const uint4 q = fragsA[(w * 3 + l) * 32 + lane];
        a[l][0] = q.x; a[l][1] = q.y; a[l][2] = q.z; a[l][3] = q.w;
    }
    const int kx0 = kx0s[w] & ~3;
    __syncthreads();
    const int z[4] = {0, 0, 0, 0}, r[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
    const int ra = 4 * (g >> 1) + (g & 1);                  // N-tile 1: n = g <-> row 4(g/2) + g%2 ; N-tile 2: + 2
    for (int it = 0; it < ITERS; ++it) {
        for (int c = 0; c < 3; ++c) {
#pragma unroll 1
            for (int r16 = 0; r16 < 40; r16 += 16) {        // 16 input rows per step (rows 32..39: half wasted, like a real 40-row patch)
                uint32_t b1[2], b2[2];
                const uint8_t* p1 = planes + plane_off(c, min(r16 + ra, 39)) + kx0 + 4 * t;
                const uint8_t* p2 = planes + plane_off(c, min(r16 + ra + 2, 39)) + kx0 + 4 * t;
                b1[0] = *(const uint32_t*)p1; b1[1] = *(const uint32_t*)(p1 + 16);
                b2[0] = *(const uint32_t*)p2; b2[1] = *(const uint32_t*)(p2 + 16);
                int d[2][3][4];
                mma_uu(d[0][0], a[0], b1, r); mma_uu(d[0][1], a[1], b1, z); mma_su(d[0][2], a[2], b1, z);
                mma_uu(d[1][0], a[0], b2, r); mma_uu(d[1][1], a[1], b2, z); mma_su(d[1][2], a[2], b2, z);
                // thread holds outputs (m = g, g+8) x rows 4t..4t+3 of this 16-row step: pack 4 rows per word
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    uint32_t v[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {            // q: row within the group of 4 = 2 * tile + (i & 1)
                        const int tile = q >> 1, i = 2 * h + (q & 1);
                        v[q] = fin(d[tile][0][i] + (d[tile][1][i] << 8) + (d[tile][2][i] << 16));
                    }
                    const uint32_t word = v[0] | (v[1] << 8) | (v[2] << 16) | (v[3] << 24);
                    mid[((r16 >> 2) + t) * MIDP + 3 * (16 * w + g + 8 * h) + c] = word;
                }
            }
        }
        __syncthreads();
    }
    out[blockIdx.x * 256 + threadIdx.x] = mid[threadIdx.x];
}

// ---- part 3b: V pass ---------------------------------------------------------------------------------------------------
// mid as above (10 row groups = 40 input rows -> K = 32 per M-tile, two k-steps would be needed beyond); 32 output rows =
// 2 M-tiles; N = 384 byte columns = 24 pairs of N-tiles; warp w takes pairs w, w+8, w+16.  Output: D[32][384] bytes.
__global__ void __launch_bounds__(256, 4) kV(int* out, const uint4* fragsA) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint32_t* mid = (uint32_t*)sm;                          // 10 * 440 words
    uint8_t* D = sm + 10 * MIDP * 4;                        // 32 x 384
    for (int i = threadIdx.x; i < 10 * MIDP; i += 256) mid[i] = i * 2654435761u;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    uint32_t a[2][3][4];
    for (int m = 0; m < 2; ++m)
        for (int l = 0; l < 3; ++l) {
            const uint4 q = fragsA[(m * 3 + l) * 32 + lane];
            a[m][l][0] = q.x; a[m][l][1] = q.y; a[m][l][2] = q.z; a[m][l][3] = q.w;
        }
    __syncthreads();
    const int z[4] = {0, 0, 0, 0}, r[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll 1
        for (int pair = w; pair < 24; pair += 8) {
            // N-tile 1: n = g <-> byte column 16 pair + 4 (g / 2) + g % 2 ; N-tile 2: + 2  (thread ends with 4 consecutive bytes)
            const int col = 16 * pair + 4 * (g >> 1) + (g & 1);
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const uint32_t* p = mid + (m * 4 + t) * MIDP + col;      // M-tile m reads row groups 4m .. 4m+7 (K = 32 rows)
                uint32_t b1[2] = {p[0], p[4 * MIDP]}, b2[2] = {p[2], p[4 * MIDP + 2]};
                int d[2][3][4];
                mma_uu(d[0][0], a[m][0], b1, r); mma_uu(d[0][1], a[m][1], b1, z); mma_su(d[0][2], a[m][2], b1, z);
                mma_uu(d[1][0], a[m][0], b2, r); mma_uu(d[1][1], a[m][1], b2, z); mma_su(d[1][2], a[m][2], b2, z);
#pragma unroll
                for (int h = 0; h < 2; ++h) {                // output rows 16 m + g + 8 h, bytes 16 pair + 4 t .. + 3
                    uint32_t v[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int tile = q >> 1, i = 2 * h + (q & 1);
                        v[q] = fin(d[tile][0][i] + (d[tile][1][i] << 8) + (d[tile][2][i] << 16));
                    }
                    *(uint32_t*)(D + (16 * m + g + 8 * h) * 384 + 16 * pair + 4 * t) = v[0] | (v[1] << 8) | (v[2] << 16) | (v[3] << 24);
                }
            }
        }
        __syncthreads();
    }
    out[blockIdx.x * 256 + threadIdx.x] = ((uint32_t*)D)[threadIdx.x];
}

static float timeit(void (*launch)(), int reps = 3) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch();
    float best = 1e9f;
    for (int i = 0; i < reps; ++i) {
        cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        best = ms < best ? ms : best;
    }
    return best;
}

static int* g_out; static uint4* g_frags; static int* g_kx0;
int main() {
    // ---- part 1 ----
    {
        std::vector<int> coef(16 * 32);
        std::vector<uint8_t> limbs(3 * 512), in(8 * 32);
        srand(7);
        for (auto& c : coef) c = (rand() % (1 << 23)) - (1 << 22) + (rand() % 3 == 0 ? 1 << 22 : 0);   // 23-bit signed, up to 2^22 + 2^22
        for (auto& c : coef) if (c >= (1 << 23)) c = (1 << 23) - 1;
        for (auto& v : in) v = rand() & 255;
        for (int i = 0; i < 512; ++i) {
            const int c = coef[i];
            limbs[i] = c & 255; limbs[512 + i] = (c >> 8) & 255; limbs[1024 + i] = (uint8_t)(int8_t)(c >> 16);
        }
        uint8_t *dA, *dI; int* dO;
        cudaMalloc(&dA, limbs.size()); cudaMalloc(&dI, in.size()); cudaMalloc(&dO, 128 * 4);
        cudaMemcpy(dA, limbs.data(), limbs.size(), cudaMemcpyHostToDevice);
        cudaMemcpy(dI, in.data(), in.size(), cudaMemcpyHostToDevice);
        probe<<<1, 32>>>(dA, dI, dO);
        std::vector<int> got(128);
        cudaMemcpy(got.data(), dO, 512, cudaMemcpyDeviceToHost);
        int bad = 0;
        for (int m = 0; m < 16; ++m)
            for (int n = 0; n < 8; ++n) {
                long long s = 1 << 21;
                for (int k = 0; k < 32; ++k) s += (long long)coef[m * 32 + k] * in[n * 32 + k];
                if ((int)s != got[m * 8 + n]) ++bad;
            }
        printf("probe: %d of 128 outputs differ from the scalar loop (%s)\n", bad, cudaGetErrorString(cudaGetLastError()));
    }
    cudaMalloc(&g_out, 132 * 4 * 256 * 4);
    cudaMalloc(&g_frags, 64 * 32 * 16); cudaMemset(g_frags, 0x11, 64 * 32 * 16);
    cudaMalloc(&g_kx0, 64); cudaMemset(g_kx0, 0, 64);
    const double clk = 1.98e9;
    // ---- part 2 ----
    {
        float ms = timeit([] { rate<<<132 * 4, 256>>>(g_out, 8); });
        const double n = 132.0 * 4 * 8 * ITERS * 16 * 8;     // warp-level MMAs
        printf("IMMA.16832 u8: %.3f ms  %.3f MMA/clk/SM  = %.0f MAC/clk/SM  (%.1f TOPS dense at 1.98 GHz)\n", ms,
               n / (ms * 1e-3 * clk) / 132, n / (ms * 1e-3 * clk) / 132 * 4096, n * 4096 * 2 / (ms * 1e-3) / 1e12);
    }
    // ---- part 3 ----
    {
        const int smH = 3 * 40 * PB + 160 + 12 * MIDP * 4;
        cudaFuncSetAttribute(kH, cudaFuncAttributeMaxDynamicSharedMemorySize, smH);
        static int s_smH; s_smH = smH;
        float ms = timeit([] { kH<<<132 * 4, 256, s_smH>>>(g_out, g_frags, g_kx0); });
        // per CTA per iter: 3 channels x 40 rows x 128 px outputs (48 rows computed, 40 valid)
        printf("H pass (IMMA): %.3f ms  %.2f output bytes/clk/SM (valid rows)  [smem %d B]  (%s)\n", ms,
               3.0 * 40 * 128 * ITERS * 4 / (ms * 1e-3 * clk), smH, cudaGetErrorString(cudaGetLastError()));
        const int smV = 10 * MIDP * 4 + 32 * 384;
        cudaFuncSetAttribute(kV, cudaFuncAttributeMaxDynamicSharedMemorySize, smV);
        static int s_smV; s_smV = smV;
        ms = timeit([] { kV<<<132 * 4, 256, s_smV>>>(g_out, g_frags); });
        printf("V pass (IMMA): %.3f ms  %.2f output bytes/clk/SM  [smem %d B]  (%s)\n", ms,
               32.0 * 384 * ITERS * 4 / (ms * 1e-3 * clk), smV, cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}
