// usdu_jpeg_decode.cu -- the data-parallel half of the baseline JPEG decode: dequantisation, the islow inverse DCT,
// fancy chroma upsampling and the YCbCr -> RGB conversion, bit for bit as PIL's open().convert("RGB") gives them with
// its bundled libjpeg-turbo.  The Huffman decode ran on the host (csrc/usdu_jpeg.cpp) and left int16 coefficient blocks.
//
// One CTA per tile: one MCU row (8 * v0 output rows) by USDU_JPEG_TILE_W output columns of one frame.
//   1. Every block the tile needs is inverse-transformed into shared memory, 8 threads per block (a column each in
//      pass 1, a row each in pass 2): the luma blocks under the tile, and the chroma blocks under it plus, for a
//      subsampled axis, the block row / column on each side (fancy upsampling reads the chroma sample beyond the
//      tile: the context rows of libjpeg's main controller).
//   2. Every output pixel takes its luma sample, its upsampled chroma samples and converts.
// The IDCT restates jidctint-avx2 / -sse2, which libjpeg-turbo runs on x86: the dequantised coefficient is the low 16
// bits of coef * quant, the sums it forms with 16-bit adds wrap, pass 1's outputs are saturated to 16 bits, pass 2's
// to 16 then 8 bits, and a block whose rows 1..7 are all zero takes the DC-only shortcut ((dc * q) << 2 in 16 bits).
// Where no intermediate leaves 16 bits this is exactly jidctint.c's arithmetic, which is what any file from a real
// encoder gives.
// Chroma edges follow jdsample.c / jdmainct.c: the sample rows above the first and below the last real row are copies
// of them, and the columns likewise; h2v1 / h2v2 upsample by replication when the chroma row is at most 2 samples wide.
#include "usdu_common.cuh"

namespace usdu {
namespace {

constexpr int kTileW = USDU_JPEG_TILE_W;
constexpr int kJThreads = 256;
constexpr int kJobs = kJThreads / 8;                // blocks transformed at once
constexpr int kCRows = 24;                          // chroma rows staged: block rows my - 1, my, my + 1
constexpr int kCCols = kTileW + 16;                 // chroma columns staged: the tile's, and one block each side

// jidctint constants (CONST_BITS = 13)
constexpr int F298 = 2446, F390 = 3196, F541 = 4433, F765 = 6270, F899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ int w16(int x) { return (int)(int16_t)(uint16_t)(uint32_t)x; }
__device__ __forceinline__ int sat16(int x) { return min(max(x, -32768), 32767); }
__device__ __forceinline__ int add(int a, int b) { return (int)((uint32_t)a + (uint32_t)b); }
__device__ __forceinline__ int sub(int a, int b) { return (int)((uint32_t)a - (uint32_t)b); }
__device__ __forceinline__ int mul(int a, int b) { return (int)((uint32_t)a * (uint32_t)b); }

// One 8-point pass over 16-bit inputs x[0..7] -> 32-bit results before the descale (pmaddwd pairs, 32-bit adds).
__device__ __forceinline__ void idct8(const int* x, int* o) {
    const int tmp2 = add(mul(x[2], F541), mul(x[6], F541 - F1847));
    const int tmp3 = add(mul(x[2], F541 + F765), mul(x[6], F541));
    const int tmp0 = mul(w16(x[0] + x[4]), 1 << 13);
    const int tmp1 = mul(w16(x[0] - x[4]), 1 << 13);
    const int t10 = add(tmp0, tmp3), t13 = sub(tmp0, tmp3), t11 = add(tmp1, tmp2), t12 = sub(tmp1, tmp2);
    const int a0 = x[7], a1 = x[5], a2 = x[3], a3 = x[1];
    const int z3 = w16(a0 + a2), z4 = w16(a1 + a3);
    const int z3p = add(mul(z3, F1175 - F1961), mul(z4, F1175));
    const int z4p = add(mul(z3, F1175), mul(z4, F1175 - F390));
    const int o0 = add(add(mul(a0, F298 - F899), mul(a3, -F899)), z3p);
    const int o3 = add(add(mul(a0, -F899), mul(a3, F1501 - F899)), z4p);
    const int o1 = add(add(mul(a1, F2053 - F2562), mul(a2, -F2562)), z4p);
    const int o2 = add(add(mul(a1, -F2562), mul(a2, F3072 - F2562)), z3p);
    o[0] = add(t10, o3), o[7] = sub(t10, o3);
    o[1] = add(t11, o2), o[6] = sub(t11, o2);
    o[2] = add(t12, o1), o[5] = sub(t12, o1);
    o[3] = add(t13, o0), o[4] = sub(t13, o0);
}

// Thread `t` (0..7) of the 8 lanes that own one block: column t in pass 1, row t in pass 2, into plane[8][pitch].
// All 32 lanes of the warp call it (active = whether this lane's group has a block).
__device__ __forceinline__ void idct_block(const int16_t* __restrict__ blk, const int32_t* __restrict__ q, int t,
                                           bool active, int16_t* ws, uint8_t* plane, int pitch) {
    int d[8];
    bool ac = false;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int c = active ? blk[r * 8 + t] : 0;
        if (r > 0) ac |= c != 0;
        d[r] = active ? w16(c * q[r * 8 + t]) : 0;
    }
    const unsigned lane = threadIdx.x & 31;
    const unsigned group = 0xFFu << (lane & ~7u);
    const bool any_ac = (__ballot_sync(0xffffffffu, ac) & group) != 0;
    if (!any_ac) {
        const int v = w16(d[0] * 4);
#pragma unroll
        for (int r = 0; r < 8; ++r) ws[r * 8 + t] = (int16_t)v;
    } else {
        int o[8];
        idct8(d, o);
#pragma unroll
        for (int r = 0; r < 8; ++r) ws[r * 8 + t] = (int16_t)sat16(add(o[r], 1 << 10) >> 11);
    }
    __syncwarp();
    int x[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = ws[t * 8 + k];
    idct8(x, o);
    if (active) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int v = min(max(sat16(add(o[k], 1 << 17) >> 18), -128), 127);
            plane[t * pitch + k] = (uint8_t)(v + 128);
        }
    }
    __syncwarp();
}

struct Job {
    const int16_t* blk;
    const int32_t* q;
    uint8_t* dst;           // top-left of the block's 8x8 in shared memory
    int pitch;
};

__global__ void __launch_bounds__(kJThreads) jpeg_decode_kernel(const uint8_t* __restrict__ src,
                                                                const int64_t* __restrict__ descs, int n,
                                                                uint8_t* __restrict__ dst) {
    __shared__ __align__(16) uint8_t ly[16 * kTileW];
    __shared__ __align__(16) uint8_t cp[2][kCRows * kCCols];
    __shared__ __align__(16) int16_t ws[kJobs][64];
    // the frame of this CTA: the last descriptor whose first CTA is <= blockIdx.x
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (descs[(int64_t)mid * USDU_JPEG_DESC_WORDS + 11] <= (int64_t)blockIdx.x) lo = mid;
        else hi = mid - 1;
    }
    const int64_t* d = descs + (int64_t)lo * USDU_JPEG_DESC_WORDS;
    const int16_t* coef = reinterpret_cast<const int16_t*>(src + d[0]);
    const int32_t* quant = reinterpret_cast<const int32_t*>(src + d[1]);
    const int W = (int)d[2], H = (int)d[3], nc = (int)d[4], h0 = (int)d[5], v0 = (int)d[6], colour = (int)d[7];
    const int mcux = (int)d[8], mcuy = (int)d[9];
    uint8_t* out = dst + d[10];
    const int tiles_x = (W + kTileW - 1) / kTileW;
    const int64_t tile = (int64_t)blockIdx.x - d[11];
    const int my = (int)(tile / tiles_x), tx = (int)(tile % tiles_x);
    if (my >= mcuy) return;
    const int x0 = tx * kTileW, y0 = my * 8 * v0;
    const int tw = min(kTileW, W - x0), th = min(8 * v0, H - y0);
    const int bw0 = mcux * h0;
    // chroma: the plane is (dh x dw) samples, blocks bw x bh = mcux x mcuy; staged from block row my - 1, column cb0
    const int dw = (W + h0 - 1) / h0, dh = (H + v0 - 1) / v0;
    const int cb0 = x0 / (8 * h0) - 1;
    const int cr0 = (v0 == 2 ? my - 1 : my), cr1 = (v0 == 2 ? my + 1 : my);               // block rows staged
    const int cc0 = (h0 == 2 ? cb0 : cb0 + 1), cc1 = min((x0 + tw - 1) / (8 * h0) + (h0 == 2), mcux - 1);
    const int ny_cols = (tw + 7) / 8;
    const int n_y = v0 * ny_cols;
    const int nr = min(cr1, mcuy - 1) - max(cr0, 0) + 1, ncc = cc1 - max(cc0, 0) + 1;
    const int n_c = nc == 3 ? 2 * nr * ncc : 0;
    const int64_t ysize = (int64_t)bw0 * mcuy * v0 * 64, csize = (int64_t)mcux * mcuy * 64;

    const int t = threadIdx.x & 7, slot = threadIdx.x >> 3;
    for (int j0 = 0; j0 < n_y + n_c; j0 += kJobs) {
        const int j = j0 + slot;
        Job job{nullptr, nullptr, nullptr, 0};
        if (j < n_y) {
            const int r = j / ny_cols, c = j % ny_cols;
            const int bx = x0 / 8 + c, by = my * v0 + r;
            job = Job{coef + ((int64_t)by * bw0 + bx) * 64, quant, ly + r * 8 * kTileW + c * 8, kTileW};
        } else if (j < n_y + n_c) {
            const int k = j - n_y, comp = k / (nr * ncc), rem = k % (nr * ncc);
            const int by = max(cr0, 0) + rem / ncc, bx = max(cc0, 0) + rem % ncc;
            job = Job{coef + ysize + comp * csize + ((int64_t)by * mcux + bx) * 64, quant + 64 * (comp + 1),
                      cp[comp] + (by - (my - 1)) * 8 * kCCols + (bx - cb0) * 8, kCCols};
        }
        idct_block(job.blk, job.q, t, job.blk != nullptr, ws[slot], job.dst, job.pitch);
    }
    __syncthreads();

    const bool fancy_h = h0 == 2 && dw > 2, fancy_v = v0 == 2 && (h0 == 1 || dw > 2);
    for (int i = threadIdx.x; i < tw * th; i += kJThreads) {
        const int py = i / tw, px = i % tw;
        const int y = y0 + py, x = x0 + px;
        const int Y = ly[py * kTileW + px];
        uint8_t* o = out + ((int64_t)y * W + x) * 3;
        if (nc == 1) {
            o[0] = o[1] = o[2] = (uint8_t)Y;
            continue;
        }
        const int rc = y / v0, cc = x / h0;
        const int lr = rc - (my - 1) * 8, lc = cc - cb0 * 8;
        int ch[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint8_t* p = cp[k];
            if (!fancy_h && !fancy_v) {
                ch[k] = p[lr * kCCols + lc];
            } else if (!fancy_v) {                                      // h2v1
                const int nb = (x & 1) ? min(cc + 1, dw - 1) : max(cc - 1, 0);
                ch[k] = (3 * p[lr * kCCols + lc] + p[lr * kCCols + nb - cb0 * 8] + ((x & 1) ? 2 : 1)) >> 2;
            } else {
                const int nbr = ((y & 1) ? min(rc + 1, dh - 1) : max(rc - 1, 0)) - (my - 1) * 8;
                if (!fancy_h) {                                         // h1v2
                    ch[k] = (3 * p[lr * kCCols + lc] + p[nbr * kCCols + lc] + ((y & 1) ? 2 : 1)) >> 2;
                } else {                                                // h2v2
                    const int nbc = ((x & 1) ? min(cc + 1, dw - 1) : max(cc - 1, 0)) - cb0 * 8;
                    const int s0 = 3 * p[lr * kCCols + lc] + p[nbr * kCCols + lc];
                    const int s1 = 3 * p[lr * kCCols + nbc] + p[nbr * kCCols + nbc];
                    ch[k] = (3 * s0 + s1 + ((x & 1) ? 7 : 8)) >> 4;
                }
            }
        }
        if (colour == USDU_JPEG_RGB) {
            o[0] = (uint8_t)Y, o[1] = (uint8_t)ch[0], o[2] = (uint8_t)ch[1];
        } else {                                                        // ycc_rgb_convert, SCALEBITS = 16
            const int cb = ch[0] - 128, cr = ch[1] - 128;
            const int r = Y + ((91881 * cr + 32768) >> 16);
            const int g = Y + ((-46802 * cr - 22554 * cb + 32768) >> 16);
            const int b = Y + ((116130 * cb + 32768) >> 16);
            o[0] = (uint8_t)min(max(r, 0), 255), o[1] = (uint8_t)min(max(g, 0), 255), o[2] = (uint8_t)min(max(b, 0), 255);
        }
    }
}

}  // namespace
}  // namespace usdu

using namespace usdu;

extern "C" {

int usdu_jpeg_decode_u8(const uint8_t* src_dev, const int64_t* descs_dev, int n, int64_t n_ctas, uint8_t* dst_dev,
                        void* stream) {
    USDU_REQUIRE(n >= 0 && n_ctas >= 0, "usdu_jpeg_decode_u8: %d frames, %lld CTAs", n, (long long)n_ctas);
    if (n == 0 || n_ctas == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && descs_dev && dst_dev, "usdu_jpeg_decode_u8: null pointer");
    USDU_REQUIRE(n_ctas <= 0x7fffffff, "usdu_jpeg_decode_u8: %lld CTAs", (long long)n_ctas);
    jpeg_decode_kernel<<<(unsigned)n_ctas, kJThreads, 0, (cudaStream_t)stream>>>(src_dev, descs_dev, n, dst_dev);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

}  // extern "C"
