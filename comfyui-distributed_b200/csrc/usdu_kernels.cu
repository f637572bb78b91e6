// usdu_kernels.cu -- sm_90a kernels of the USDU tile path and their C-ABI launchers.
//
// All pixel arithmetic is integer and bit-exact with the reference's Pillow path
// (specs V1-V5 in SURVEY.md section 8a, restated in oracle/usdu_oracle.py):
//   Q0/Q1   trunc(255*x)                         utils/image.py:8-10
//   K2      crop + LANCZOS (H pass, u8, V pass)  upscale/tile_ops.py:96-155
//   K3      rectangle + 3x3 box "Gaussian"       upscale/tile_ops.py:289-308
//   K4      LANCZOS back + integer composite     upscale/tile_ops.py:310-349
// These kernels are HBM-bandwidth bound byte/integer work: no tensor cores.
#include "usdu_common.cuh"

namespace usdu {

// ======================================================================================
// Q0 / dequantise / Q1
// ======================================================================================
// One thread produces 16 canvas bytes (one uint4 store) from 16 floats (4 x float4 loads).
__device__ __forceinline__ void
quantize_rows_body(const float* __restrict__ img, uint8_t* __restrict__ canvas, int rows, int W3,
                   int64_t pitch, int vec_ok, int H, int y0, int n_rows) {
    // logical row i of `rows` = B * n_rows  ->  physical row b * H + y0 + (i % n_rows)
    const int chunks = (W3 + 15) >> 4;
    const int64_t total = (int64_t)rows * chunks;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t lrow = i / chunks;
        const int j0 = (int)(i - lrow * chunks) << 4;
        const int64_t fb = lrow / n_rows;
        const int64_t row = fb * H + y0 + (lrow - fb * n_rows);
        const float* src = img + row * W3 + j0;
        uint8_t* dst = canvas + row * pitch + j0;
        if (vec_ok && j0 + 16 <= W3) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4 a = __ldcs(s4), b = __ldcs(s4 + 1), c = __ldcs(s4 + 2), d = __ldcs(s4 + 3);
            uint4 o;
            o.x = quant_u8(a.x) | (quant_u8(a.y) << 8) | (quant_u8(a.z) << 16) | (quant_u8(a.w) << 24);
            o.y = quant_u8(b.x) | (quant_u8(b.y) << 8) | (quant_u8(b.z) << 16) | (quant_u8(b.w) << 24);
            o.z = quant_u8(c.x) | (quant_u8(c.y) << 8) | (quant_u8(c.z) << 16) | (quant_u8(c.w) << 24);
            o.w = quant_u8(d.x) | (quant_u8(d.y) << 8) | (quant_u8(d.z) << 16) | (quant_u8(d.w) << 24);
            *reinterpret_cast<uint4*>(dst) = o;
        } else {
            const int n = min(16, W3 - j0);
            for (int k = 0; k < n; ++k) dst[k] = (uint8_t)quant_u8(src[k]);
        }
    }
}

__global__ void __launch_bounds__(kThreads)
quantize_canvas_kernel(const float* __restrict__ img, uint8_t* __restrict__ canvas, int rows, int W3,
                       int64_t pitch, int vec_ok, int H, int y0, int n_rows) {
    quantize_rows_body(img, canvas, rows, W3, pitch, vec_ok, H, y0, n_rows);
}

// One thread turns ONE canvas word (4 bytes) into one float4: consecutive lanes read consecutive
// words (128 B per warp load) and write consecutive float4 (512 B per warp store, every 32-byte
// sector written whole by one instruction).  Rows on blockIdx.y, no integer division.
__device__ __forceinline__ void
dequantize_rows_body(const uint8_t* __restrict__ canvas, float* __restrict__ img, int rows, int W3,
                     int64_t pitch, int vec_ok, int H, int y0, int n_rows) {
    if (vec_ok) {
        const int words = W3 >> 2;
        for (int lrow = blockIdx.y; lrow < rows; lrow += gridDim.y) {
            const int fb = lrow / n_rows;
            const int64_t row = (int64_t)fb * H + y0 + (lrow - fb * n_rows);
            const uint32_t* src = reinterpret_cast<const uint32_t*>(canvas + (int64_t)row * pitch);
            float4* dst = reinterpret_cast<float4*>(img + (int64_t)row * W3);
#pragma unroll 4
            for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) {
                const uint32_t v = __ldcs(src + w);
                float4 o;
                o.x = dequant_u8_fast(v & 0xFF);
                o.y = dequant_u8_fast((v >> 8) & 0xFF);
                o.z = dequant_u8_fast((v >> 16) & 0xFF);
                o.w = dequant_u8_fast(v >> 24);
                __stcs(dst + w, o);
            }
        }
        return;
    }
    for (int lrow = blockIdx.y; lrow < rows; lrow += gridDim.y) {
        const int fb = lrow / n_rows;
        const int64_t row = (int64_t)fb * H + y0 + (lrow - fb * n_rows);
        const uint8_t* src = canvas + row * pitch;
        float* dst = img + row * W3;
        for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < W3; j += gridDim.x * blockDim.x) dst[j] = dequant_u8_fast(src[j]);
    }
}

__global__ void __launch_bounds__(kThreads)
dequantize_canvas_kernel(const uint8_t* __restrict__ canvas, float* __restrict__ img, int rows, int W3,
                         int64_t pitch, int vec_ok, int H, int y0, int n_rows) {
    dequantize_rows_body(canvas, img, rows, W3, pitch, vec_ok, H, y0, n_rows);
}

// The same two passes for a captured graph that runs them in row bands beside the wave loop (engine.run_split): the fp32
// image / result address comes from a device-side usdu_stream_args block the host rewrites before every replay, and the
// grid is a few persistent CTAs that stride over the band, so the pass holds few of the CTA slots the wave kernels need.
// Both are launched only for 16-byte aligned pointers and widths that are multiples of 4 (the vector path).
__global__ void __launch_bounds__(kThreads)
quantize_rows_streamed_kernel(const usdu_stream_args* __restrict__ args, uint8_t* __restrict__ canvas, int rows, int W3,
                              int64_t pitch, int H, int y0, int n_rows) {
    quantize_rows_body(args->img_dev, canvas, rows, W3, pitch, 1, H, y0, n_rows);
}

__global__ void __launch_bounds__(kThreads)
dequantize_rows_streamed_kernel(const uint8_t* __restrict__ canvas, const usdu_stream_args* __restrict__ args, int rows, int W3,
                                int64_t pitch, int H, int y0, int n_rows) {
    dequantize_rows_body(canvas, args->out_dev, rows, W3, pitch, 1, H, y0, n_rows);
}

// The master's gather of a multi-GPU job: canvas rows [y[q], y[q+1]) come from slab q's canvas (base[q] -- a peer's HBM
// mapped over NVLink, or the local one), every row is dequantised into the local fp32 result.  A CTA moves 4 KB of a row:
// 16-byte loads (few, wide requests on the link), a shared-memory turn, whole-sector float4 stores.
struct GatherArgs {
    const uint8_t* base[USDU_MAX_SLABS];
    int y[USDU_MAX_SLABS + 1];
    int n;
};

__global__ void __launch_bounds__(kThreads)
gather_dequantize_kernel(GatherArgs a, float* __restrict__ img, int rows_total, int H, int W3, int64_t pitch) {
    __shared__ uint4 stage[kThreads];
    const int c0 = blockIdx.x * (kThreads * 16);                 // first byte of this CTA's chunk of the row
    for (int lrow = blockIdx.y; lrow < rows_total; lrow += gridDim.y) {
        const int fb = lrow / H, yy = lrow - fb * H;
        int q = 0;
        while (q + 1 < a.n && yy >= a.y[q + 1]) ++q;
        const uint8_t* src = a.base[q] + ((int64_t)fb * H + yy) * pitch + c0;
        const int off = threadIdx.x * 16;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (c0 + off + 16 <= W3) v = __ldcs(reinterpret_cast<const uint4*>(src + off));
        else if (c0 + off < W3) {                                 // row tail (W3 % 16 != 0): word loads, W3 % 4 == 0
            uint32_t w[4] = {0, 0, 0, 0};
            for (int k = 0; k < 4; ++k) if (c0 + off + 4 * k < W3) w[k] = __ldcs(reinterpret_cast<const uint32_t*>(src + off) + k);
            v = make_uint4(w[0], w[1], w[2], w[3]);
        }
        __syncthreads();                                          // the previous row's readers are done
        stage[threadIdx.x] = v;
        __syncthreads();
        float4* dst = reinterpret_cast<float4*>(img + ((int64_t)fb * H + yy) * W3 + c0);
        const uint32_t* words = reinterpret_cast<const uint32_t*>(stage);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int wi = k * kThreads + threadIdx.x;            // consecutive lanes -> consecutive float4
            if (c0 + 4 * wi < W3) {
                const uint32_t u = words[wi];
                float4 o;
                o.x = dequant_u8_fast(u & 0xFF); o.y = dequant_u8_fast((u >> 8) & 0xFF);
                o.z = dequant_u8_fast((u >> 16) & 0xFF); o.w = dequant_u8_fast(u >> 24);
                __stcs(dst + wi, o);
            }
        }
    }
}

// ... and the all-gather of the quantised INPUT slabs (host path: every rank uploads and quantises 1/N of the rows, then
// pulls the other N-1 slabs into its own working canvas): the same walk, bytes copied as they are, 16 per thread.
__global__ void __launch_bounds__(kThreads)
gather_canvas_kernel(GatherArgs a, uint8_t* __restrict__ dst, int rows_total, int H, int row_bytes, int64_t pitch) {
    const int off = (blockIdx.x * kThreads + threadIdx.x) * 16;
    if (off >= row_bytes) return;
    for (int lrow = blockIdx.y; lrow < rows_total; lrow += gridDim.y) {
        const int fb = lrow / H, yy = lrow - fb * H;
        int q = 0;
        while (q + 1 < a.n && yy >= a.y[q + 1]) ++q;
        const int64_t at = ((int64_t)fb * H + yy) * pitch + off;
        if (a.base[q] == dst) continue;                            // this rank's own slab is already in place
        *reinterpret_cast<uint4*>(dst + at) = __ldcs(reinterpret_cast<const uint4*>(a.base[q] + at));
    }
}

__global__ void __launch_bounds__(kThreads)
pack_u8_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, int64_t n) {
    const int64_t n16 = n >> 4;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = tid; i < n16; i += stride) {
        const float4* s4 = reinterpret_cast<const float4*>(src) + i * 4;
        float4 a = __ldcs(s4), b = __ldcs(s4 + 1), c = __ldcs(s4 + 2), d = __ldcs(s4 + 3);
        uint4 o;
        o.x = quant_u8(a.x) | (quant_u8(a.y) << 8) | (quant_u8(a.z) << 16) | (quant_u8(a.w) << 24);
        o.y = quant_u8(b.x) | (quant_u8(b.y) << 8) | (quant_u8(b.z) << 16) | (quant_u8(b.w) << 24);
        o.z = quant_u8(c.x) | (quant_u8(c.y) << 8) | (quant_u8(c.z) << 16) | (quant_u8(c.w) << 24);
        o.w = quant_u8(d.x) | (quant_u8(d.y) << 8) | (quant_u8(d.z) << 16) | (quant_u8(d.w) << 24);
        reinterpret_cast<uint4*>(dst)[i] = o;
    }
    for (int64_t i = (n16 << 4) + tid; i < n; i += stride) dst[i] = (uint8_t)quant_u8(src[i]);
}

__global__ void __launch_bounds__(kThreads)
unpack_f32_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int64_t n) {
    __shared__ float lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = dequant_u8(i);
    __syncthreads();
    const int64_t n16 = n >> 4;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = tid; i < n16; i += stride) {
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(src) + i);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        float4* d4 = reinterpret_cast<float4*>(dst) + i * 4;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float4 o;
            o.x = lut[w[k] & 0xFF];
            o.y = lut[(w[k] >> 8) & 0xFF];
            o.z = lut[(w[k] >> 16) & 0xFF];
            o.w = lut[w[k] >> 24];
            d4[k] = o;
        }
    }
    for (int64_t i = (n16 << 4) + tid; i < n; i += stride) dst[i] = lut[src[i]];
}

// The T0 sampler stand-in of the tests / benchmark as ONE pass: out = clamp(x*omd + nd, 0, 1),
// every step individually rounded (no FMA contraction) so that it equals the oracle's numpy.
__global__ void __launch_bounds__(kThreads)
t0_denoise_kernel(const float4* __restrict__ x, const float4* __restrict__ nd, float4* __restrict__ out,
                  int64_t n4, int64_t frame4, float omd) {
    pdl_launch_dependents();
    pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 a = __ldcs(x + i);
        const float4 b = __ldg(nd + (i % frame4));
        float4 o;
        o.x = fminf(fmaxf(__fadd_rn(__fmul_rn(a.x, omd), b.x), 0.0f), 1.0f);
        o.y = fminf(fmaxf(__fadd_rn(__fmul_rn(a.y, omd), b.y), 0.0f), 1.0f);
        o.z = fminf(fmaxf(__fadd_rn(__fmul_rn(a.z, omd), b.z), 0.0f), 1.0f);
        o.w = fminf(fmaxf(__fadd_rn(__fmul_rn(a.w, omd), b.w), 0.0f), 1.0f);
        out[i] = o;
    }
}

// ======================================================================================
// shared building blocks of the two resampling kernels
// ======================================================================================
// Input index range [lo, hi) that outputs [o0, o0+cnt) of an axis read.
__device__ __forceinline__ void axis_range(const int32_t* tabs, int tab, int o0, int cnt, int& lo, int& hi) {
    if (tab < 0) {
        lo = o0;
        hi = o0 + cnt;
    } else {
        const int32_t* b = tabs + tab + USDU_TAB_HEADER;
        lo = b[2 * o0];
        hi = b[2 * (o0 + cnt - 1)] + b[2 * (o0 + cnt - 1) + 1];
    }
}

// A source byte of the horizontal pass: u8 as it is, fp32 through the truncating cast Q1.
__device__ __forceinline__ uint32_t load8(const uint8_t* p) { return *p; }
__device__ __forceinline__ uint32_t load8(const float* p) { return quant_u8(__ldg(p)); }

// Horizontal pass: in[rows][in_pitch] (u8 or fp32, pixel-interleaved, column 0 == input pixel ix0; the patch staged in
// shared memory, or the source itself in global memory) -> mid[rows][mid_pitch] holding `ow` output pixels starting at
// output index ox0.
template <typename T>
__device__ __forceinline__ void hpass(const T* in, int64_t in_pitch, int ix0, uint8_t* mid, int mid_pitch,
                                      int rows, int ox0, int ow, const int32_t* tabs, int tab) {
    const int ow3 = ow * 3;
    if (tab < 0) {
        for (int i = threadIdx.x; i < rows * ow3; i += blockDim.x) {
            const int r = i / ow3, j = i - r * ow3;
            mid[r * mid_pitch + j] = (uint8_t)load8(in + r * in_pitch + j);
        }
        return;
    }
    const TableView t = table_at(tabs, tab);
    for (int i = threadIdx.x; i < rows * ow; i += blockDim.x) {
        const int r = i / ow, xx = i - r * ow;
        const int xmin = __ldg(t.bounds + 2 * (ox0 + xx));
        const int n = __ldg(t.bounds + 2 * (ox0 + xx) + 1);
        const int32_t* k = t.kk + (int64_t)(ox0 + xx) * t.ksize;
        const T* p = in + r * in_pitch + (xmin - ix0) * 3;
        int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
        for (int q = 0; q < n; ++q) {
            const int kv = __ldg(k + q);
            a0 += (int)load8(p + 3 * q) * kv;
            a1 += (int)load8(p + 3 * q + 1) * kv;
            a2 += (int)load8(p + 3 * q + 2) * kv;
        }
        uint8_t* o = mid + r * mid_pitch + xx * 3;
        o[0] = (uint8_t)clip8(a0 >> kPrecisionBits);
        o[1] = (uint8_t)clip8(a1 >> kPrecisionBits);
        o[2] = (uint8_t)clip8(a2 >> kPrecisionBits);
    }
}

// Vertical pass value for output row index oy (absolute) and byte column j of mid.
__device__ __forceinline__ uint32_t vpass_at(const uint8_t* mid, int mid_pitch, int iy0, int oy, int j,
                                             const TableView& t) {
    const int ymin = __ldg(t.bounds + 2 * oy);
    const int n = __ldg(t.bounds + 2 * oy + 1);
    const int32_t* k = t.kk + (int64_t)oy * t.ksize;
    const uint8_t* p = mid + (ymin - iy0) * mid_pitch + j;
    int acc = 1 << (kPrecisionBits - 1);
    for (int q = 0; q < n; ++q) acc += p[q * mid_pitch] * __ldg(k + q);
    return clip8(acc >> kPrecisionBits);
}

// ======================================================================================
// K2: crop + LANCZOS resize -> fp32 tile
// ======================================================================================
__global__ void __launch_bounds__(kThreads)
crop_resize_kernel(const uint8_t* __restrict__ canvas, int H, int W, int64_t pitch,
                   const int32_t* __restrict__ tiles, const int32_t* __restrict__ tabs,
                   const int32_t* __restrict__ items, float* __restrict__ out, int in_pitch, int max_rows, int blk_w, int blk_h) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int32_t* it = items + (int64_t)blockIdx.x * USDU_CROP_ITEM_WORDS;
    const int32_t* T = tiles + (int64_t)it[0] * USDU_TILE_WORDS;
    const int b = blockIdx.y;
    const int ox0 = it[1], oy0 = it[2];
    const int64_t out_off = (int64_t)(uint32_t)it[3] | ((int64_t)it[4] << 32);
    const int x1 = T[USDU_T_X1], y1 = T[USDU_T_Y1];
    const int pw = T[USDU_T_PW], ph = T[USDU_T_PH];
    const int tabH = T[USDU_T_TAB_CROP_H], tabV = T[USDU_T_TAB_CROP_V];
    const int ow = min(blk_w, pw - ox0), oh = min(blk_h, ph - oy0);
    int ix0, ix1, iy0, iy1;
    axis_range(tabs, tabH, ox0, ow, ix0, ix1);
    axis_range(tabs, tabV, oy0, oh, iy0, iy1);
    const int rows = iy1 - iy0, cols3 = (ix1 - ix0) * 3;
    uint8_t* in = smem;
    const int mid_pitch = BW * 3;
    uint8_t* mid = smem + (size_t)max_rows * in_pitch;

    // stage the crop-window patch (u8) from the canvas
    const uint8_t* src = canvas + ((int64_t)b * H + (y1 + iy0)) * pitch + (int64_t)(x1 + ix0) * 3;
    for (int i = threadIdx.x; i < rows * cols3; i += blockDim.x) {
        const int r = i / cols3, j = i - r * cols3;
        in[r * in_pitch + j] = src[(int64_t)r * pitch + j];
    }
    __syncthreads();
    hpass(in, in_pitch, ix0, mid, mid_pitch, rows, ox0, ow, tabs, tabH);
    __syncthreads();
    const int ow3 = ow * 3;
    float* dst = out + out_off + ((int64_t)b * ph + oy0) * pw * 3 + (int64_t)ox0 * 3;
    if (tabV < 0) {
        for (int i = threadIdx.x; i < oh * ow3; i += blockDim.x) {
            const int yy = i / ow3, j = i - yy * ow3;
            dst[(int64_t)yy * pw * 3 + j] = dequant_u8(mid[yy * mid_pitch + j]);
        }
    } else {
        const TableView tv = table_at(tabs, tabV);
        for (int i = threadIdx.x; i < oh * ow3; i += blockDim.x) {
            const int yy = i / ow3, j = i - yy * ow3;
            dst[(int64_t)yy * pw * 3 + j] = dequant_u8(vpass_at(mid, mid_pitch, iy0, oy0 + yy, j, tv));
        }
    }
}

// ======================================================================================
// K4: quantise + LANCZOS back + integer alpha composite, per canvas block
// ======================================================================================
// kDirect: the patch of the processed tile a block reads would not fit in shared memory (a canvas far smaller than the
// tile: 2304 -> 64 px back-resizes 324 x 324 pixels into a 4 x 4 block); the horizontal pass then reads (and quantises)
// the tile in global memory and only the intermediate [max_rows][blk_w*3] is staged.
template <bool kSrcU8, bool kDirect>
__global__ void __launch_bounds__(kThreads)
blend_kernel(uint8_t* __restrict__ canvas, int H, int W, int64_t pitch, const int32_t* __restrict__ tiles,
             const int32_t* __restrict__ tabs, const uint8_t* __restrict__ mask_pool,
             const int32_t* __restrict__ items, const int32_t* __restrict__ cover,
             const void* __restrict__ src_v, int in_pitch, int max_rows, int blk_w, int blk_h) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int32_t* it = items + (int64_t)blockIdx.x * USDU_BLEND_ITEM_WORDS;
    const int b = blockIdx.y;
    const int bx0 = it[0], by0 = it[1];
    const int bw = min(blk_w, W - bx0), bh = min(blk_h, H - by0);
    const int d_pitch = BW * 3;
    const int mid_pitch = blk_w * 3;
    uint8_t* D = smem;                                // [BH][BW*3] canvas block
    uint8_t* mid = D + BH * d_pitch;                  // [max_rows][blk_w*3]
    uint8_t* in = mid + (size_t)max_rows * mid_pitch; // [max_rows][in_pitch] (staged path)

    uint8_t* cblk = canvas + ((int64_t)b * H + by0) * pitch + (int64_t)bx0 * 3;
    const int bw3 = bw * 3;
    for (int i = threadIdx.x; i < bh * bw3; i += blockDim.x) {
        const int r = i / bw3, j = i - r * bw3;
        D[r * d_pitch + j] = cblk[(int64_t)r * pitch + j];
    }
    const int c0 = it[2], cn = it[3];
    for (int e = 0; e < cn; ++e) {
        const int32_t* C = cover + (int64_t)(c0 + e) * USDU_COVER_WORDS;
        const int32_t* T = tiles + (int64_t)C[0] * USDU_TILE_WORDS;
        const int64_t src_off = (int64_t)(uint32_t)C[1] | ((int64_t)C[2] << 32);
        const int x1 = T[USDU_T_X1], y1 = T[USDU_T_Y1], ew = T[USDU_T_EW], eh = T[USDU_T_EH];
        const int pw = T[USDU_T_PW], ph = T[USDU_T_PH];
        // block  ∩  crop window  ∩  support of the feather template (alpha == 0 outside it)
        const int X0 = max(bx0, x1 + T[USDU_T_SUP_X0]), X1 = min(bx0 + bw, x1 + T[USDU_T_SUP_X1]);
        const int Y0 = max(by0, y1 + T[USDU_T_SUP_Y0]), Y1 = min(by0 + bh, y1 + T[USDU_T_SUP_Y1]);
        if (X1 <= X0 || Y1 <= Y0) continue;  // uniform across the block
        const int ox0 = X0 - x1, ow = X1 - X0, oy0 = Y0 - y1, oh = Y1 - Y0;
        const int tabH = T[USDU_T_TAB_BLEND_H], tabV = T[USDU_T_TAB_BLEND_V];
        int ix0, ix1, iy0, iy1;
        axis_range(tabs, tabH, ox0, ow, ix0, ix1);
        axis_range(tabs, tabV, oy0, oh, iy0, iy1);
        const int rows = iy1 - iy0, cols3 = (ix1 - ix0) * 3;
        __syncthreads();  // previous tile's composite (and the D load) done before in/mid are reused
        const int64_t frame = (int64_t)ph * pw * 3;
        const int64_t s_off = src_off + b * frame + ((int64_t)iy0 * pw + ix0) * 3;
        if (kDirect) {
            if (kSrcU8)
                hpass(static_cast<const uint8_t*>(src_v) + s_off, (int64_t)pw * 3, ix0, mid, mid_pitch, rows, ox0, ow, tabs, tabH);
            else
                hpass(static_cast<const float*>(src_v) + s_off, (int64_t)pw * 3, ix0, mid, mid_pitch, rows, ox0, ow, tabs, tabH);
        } else {
            // stage the processed-tile patch, quantised to u8 (Q1)
            if (kSrcU8) {
                const uint8_t* s = static_cast<const uint8_t*>(src_v) + s_off;
                for (int i = threadIdx.x; i < rows * cols3; i += blockDim.x) {
                    const int r = i / cols3, j = i - r * cols3;
                    in[r * in_pitch + j] = s[(int64_t)r * pw * 3 + j];
                }
            } else {
                const float* s = static_cast<const float*>(src_v) + s_off;
                for (int i = threadIdx.x; i < rows * cols3; i += blockDim.x) {
                    const int r = i / cols3, j = i - r * cols3;
                    in[r * in_pitch + j] = (uint8_t)quant_u8(__ldg(s + (int64_t)r * pw * 3 + j));
                }
            }
            __syncthreads();
            hpass(in, in_pitch, ix0, mid, mid_pitch, rows, ox0, ow, tabs, tabH);
        }
        __syncthreads();
        const uint8_t* mk = mask_pool + (int64_t)(uint32_t)T[USDU_T_MASK_OFF] +
                            (int64_t)oy0 * T[USDU_T_MASK_PITCH] + ox0;
        const int mpitch = T[USDU_T_MASK_PITCH];
        uint8_t* Dw = D + (Y0 - by0) * d_pitch + (X0 - bx0) * 3;
        const int ow3 = ow * 3;
        TableView tv;
        if (tabV >= 0) tv = table_at(tabs, tabV);
        for (int i = threadIdx.x; i < oh * ow3; i += blockDim.x) {
            const int yy = i / ow3, j = i - yy * ow3;
            const uint32_t S = (tabV < 0) ? mid[yy * mid_pitch + j]
                                          : vpass_at(mid, mid_pitch, iy0, oy0 + yy, j, tv);
            const uint32_t A = __ldg(mk + (int64_t)yy * mpitch + j / 3);
            uint8_t* d = Dw + yy * d_pitch + j;
            *d = (uint8_t)composite8(S, *d, A);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < bh * bw3; i += blockDim.x) {
        const int r = i / bw3, j = i - r * bw3;
        cblk[(int64_t)r * pitch + j] = D[r * d_pitch + j];
    }
}

// ======================================================================================
// K3: feather templates
// ======================================================================================
// One extended-box pass over a line in shared memory, edge-replicated at the CANVAS
// borders [0, n_canvas); the line holds canvas positions [lo, lo+len).  Reads that fall
// outside the held range (but inside the canvas) are clamped to the held range: they
// only influence outputs outside the window (see usdu_build_feather_masks).
__device__ __forceinline__ void box_pass(const uint8_t* src, uint8_t* dst, int len, int lo, int n_canvas,
                                         int rad, uint32_t ww, uint32_t fw) {
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        const int pos = lo + i;
        uint32_t acc = 0;
        for (int d = -rad; d <= rad; ++d) {
            int p = min(max(pos + d, 0), n_canvas - 1) - lo;
            p = min(max(p, 0), len - 1);
            acc += src[p];
        }
        int pl = min(max(pos - rad - 1, 0), n_canvas - 1) - lo;
        int pr = min(max(pos + rad + 1, 0), n_canvas - 1) - lo;
        pl = min(max(pl, 0), len - 1);
        pr = min(max(pr, 0), len - 1);
        const uint32_t bulk = acc * ww + (uint32_t)(src[pl] + src[pr]) * fw;
        dst[i] = (uint8_t)((bulk + (1u << 23)) >> 24);
    }
}

struct MaskSpecDev {
    int W, H, bx1, by1, bx2, by2, x1, y1, x2, y2;
    int rad;
    uint32_t ww, fw;
    int blur;
    int64_t out_off;
    int out_pitch;
    int64_t scratch_off;  // hx[ew] then vt[256][eh]
};

// blocks 0..255: vertical profile of amplitude blockIdx.x over [y1,y2); block 256: hx over [x1,x2)
__global__ void __launch_bounds__(kThreads)
mask_profiles_kernel(const MaskSpecDev* __restrict__ specs, uint8_t* __restrict__ scratch, int max_len) {
    extern __shared__ __align__(16) uint8_t smem[];
    const MaskSpecDev s = specs[blockIdx.y];
    const bool horiz = blockIdx.x == 256;
    const int amp = horiz ? 255 : blockIdx.x;
    const int n_canvas = horiz ? s.W : s.H;
    const int r0 = horiz ? s.bx1 : s.by1, r1 = horiz ? s.bx2 : s.by2;
    const int w0 = horiz ? s.x1 : s.y1, w1 = horiz ? s.x2 : s.y2;
    const int ext = 3 * (s.rad + 1);
    const int lo = max(0, w0 - ext), hi = min(n_canvas, w1 + ext);
    const int len = hi - lo;
    uint8_t* a = smem;
    uint8_t* bbuf = smem + max_len;
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        const int pos = lo + i;
        a[i] = (pos >= r0 && pos < r1) ? (uint8_t)amp : 0;
    }
    __syncthreads();
    if (s.blur > 0) {
        box_pass(a, bbuf, len, lo, n_canvas, s.rad, s.ww, s.fw);
        __syncthreads();
        box_pass(bbuf, a, len, lo, n_canvas, s.rad, s.ww, s.fw);
        __syncthreads();
        box_pass(a, bbuf, len, lo, n_canvas, s.rad, s.ww, s.fw);
        __syncthreads();
    } else {
        bbuf = a;
    }
    const int ew = s.x2 - s.x1, eh = s.y2 - s.y1;
    uint8_t* dst = scratch + s.scratch_off + (horiz ? 0 : (int64_t)ew + (int64_t)amp * eh);
    const int cnt = w1 - w0;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) dst[i] = bbuf[w0 - lo + i];
}

__global__ void __launch_bounds__(kThreads)
mask_expand_kernel(const MaskSpecDev* __restrict__ specs, const uint8_t* __restrict__ scratch,
                   uint8_t* __restrict__ pool) {
    const MaskSpecDev s = specs[blockIdx.y];
    const int ew = s.x2 - s.x1, eh = s.y2 - s.y1;
    const uint8_t* hx = scratch + s.scratch_off;
    const uint8_t* vt = hx + ew;
    uint8_t* out = pool + s.out_off;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ew * eh; i += gridDim.x * blockDim.x) {
        const int y = i / ew, x = i - y * ew;
        out[(int64_t)y * s.out_pitch + x] = vt[(int64_t)hx[x] * eh + y];
    }
}

static inline int grid_for(int64_t blocks) {
    const int64_t cap = (int64_t)grid_sms() * 16;
    return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

constexpr size_t kMaxSmem = 227 * 1024;   // dynamic shared memory a CTA may opt in to on sm_90

static int smem_optin(const void* fn, size_t bytes) {
    if (bytes > kMaxSmem) {
        set_error("kernel needs %zu bytes of shared memory (> 227 KB): patch too large", bytes);
        return USDU_ERR_UNSUPPORTED;
    }
    return raise_smem_limit(fn, bytes);
}

}  // namespace usdu

namespace usdu { namespace fast {
int launch_crop(const uint8_t* canvas, int B, int H, int W, int64_t pitch, const int32_t* tiles, const int32_t* tabs,
                const int32_t* items, int n_items, int patch_w, int patch_h, float* out, cudaStream_t st);
int launch_blend(uint8_t* canvas, int B, int H, int W, int64_t pitch, const int32_t* tiles, const int32_t* tabs,
                 const uint8_t* mask_pool, const int32_t* items, int n_items, const int32_t* cover, int patch_w,
                 int patch_h, const void* src, int src_is_u8, int block_rows, int remote, cudaStream_t st);
} }

namespace usdu { namespace mma {
int launch_crop(const void* canvas, int src_f32, int B, int H, int W, int64_t pitch, const int32_t* tabs, const int32_t* items,
                int n_items, int patch_w, int patch_h, float* out, int two_ksteps, cudaStream_t st);
int launch_blend(uint8_t* canvas, int B, int H, int W, int64_t pitch, const int32_t* tabs, const uint8_t* mask_pool,
                 const int32_t* items, int n_items, int patch_w, int patch_h, const void* src, int src_is_u8, int block_rows,
                 int two_ksteps, cudaStream_t st);
} }

using namespace usdu;

extern "C" {

int usdu_quantize_rows(const float* img_dev, uint8_t* canvas_dev, int B, int H, int W, int64_t pitch, int y0, int y1,
                       void* stream) {
    USDU_REQUIRE(img_dev && canvas_dev, "usdu_quantize_rows: null pointer");
    USDU_REQUIRE(B > 0 && H > 0 && W > 0, "usdu_quantize_rows: bad shape %dx%dx%d", B, H, W);
    USDU_REQUIRE(0 <= y0 && y0 <= y1 && y1 <= H, "usdu_quantize_rows: bad row range [%d, %d) of %d", y0, y1, H);
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0, "usdu_quantize_rows: pitch %lld must be >= 3*W and a multiple of 16", (long long)pitch);
    if (y1 == y0) return USDU_OK;
    const int W3 = W * 3;
    const int vec_ok = (W3 % 4 == 0) && (((uintptr_t)img_dev & 15) == 0) && (((uintptr_t)canvas_dev & 15) == 0);
    const int64_t total = (int64_t)B * (y1 - y0) * ((W3 + 15) / 16);
    // short-lived CTAs (up to 128 per SM, ~1 trip each on the 8K canvas); the pass that runs beside the wave kernels is
    // usdu_quantize_rows_streamed, with a few persistent CTAs instead
    const int64_t qblocks = (total + kThreads - 1) / kThreads;
    const int64_t qcap = (int64_t)grid_sms() * 128;
    const int grid = (int)(qblocks < 1 ? 1 : (qblocks > qcap ? qcap : qblocks));
    quantize_canvas_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(img_dev, canvas_dev, B * (y1 - y0), W3, pitch, vec_ok, H, y0, y1 - y0);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_quantize_canvas(const float* img_dev, uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                         void* stream) {
    USDU_REQUIRE(H > 0, "usdu_quantize_canvas: bad shape %dx%dx%d", B, H, W);
    return usdu_quantize_rows(img_dev, canvas_dev, B, H, W, pitch, 0, H, stream);
}

int usdu_dequantize_rows(const uint8_t* canvas_dev, float* img_dev, int B, int H, int W, int64_t pitch, int y0, int y1,
                         void* stream) {
    USDU_REQUIRE(img_dev && canvas_dev, "usdu_dequantize_rows: null pointer");
    USDU_REQUIRE(B > 0 && H > 0 && W > 0, "usdu_dequantize_rows: bad shape %dx%dx%d", B, H, W);
    USDU_REQUIRE(0 <= y0 && y0 <= y1 && y1 <= H, "usdu_dequantize_rows: bad row range [%d, %d) of %d", y0, y1, H);
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0, "usdu_dequantize_rows: pitch %lld must be >= 3*W and a multiple of 16", (long long)pitch);
    if (y1 == y0) return USDU_OK;
    const int W3 = W * 3;
    const int vec_ok = (W3 % 4 == 0) && (((uintptr_t)img_dev & 15) == 0) && (((uintptr_t)canvas_dev & 15) == 0);
    const int per_row = vec_ok ? W3 / 4 : W3;
    int gx = (per_row + kThreads * 4 - 1) / (kThreads * 4);          // ~4 items per thread along a row
    if (gx < 1) gx = 1;
    int64_t gy = (int64_t)B * (y1 - y0);
    if (gy > 65535) gy = 65535;
    const int64_t qcap = (int64_t)grid_sms() * 128;                 // short-lived CTAs, see usdu_quantize_rows
    if (gy * gx > qcap) gy = (qcap + gx - 1) / gx;
    if (gy < 1) gy = 1;
    dequantize_canvas_kernel<<<dim3(gx, (unsigned)gy), kThreads, 0, (cudaStream_t)stream>>>(canvas_dev, img_dev, B * (y1 - y0), W3, pitch, vec_ok, H, y0, y1 - y0);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_stream_args_set(usdu_stream_args* args_dev, const float* img_dev, float* out_dev, void* stream) {
    USDU_REQUIRE(args_dev && img_dev && out_dev, "usdu_stream_args_set: null pointer");
    USDU_REQUIRE((((uintptr_t)args_dev | (uintptr_t)img_dev | (uintptr_t)out_dev) & 15) == 0,
                 "usdu_stream_args_set: the block, the image and the result must be 16-byte aligned");
    const usdu_stream_args host = {img_dev, out_dev};    // pageable: the driver stages it before cudaMemcpyAsync returns
    USDU_CUDA(cudaMemcpyAsync(args_dev, &host, sizeof(host), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return USDU_OK;
}

// Grid of a streamed pass: at most max_ctas CTAs, each a persistent grid-stride loop over the band.
static int check_streamed(const char* what, const void* args_dev, const uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                          int y0, int y1, int max_ctas) {
    USDU_REQUIRE(args_dev && canvas_dev, "%s: null pointer", what);
    USDU_REQUIRE(B > 0 && H > 0 && W > 0 && W % 4 == 0, "%s: bad shape %dx%dx%d (W must be a multiple of 4)", what, B, H, W);
    USDU_REQUIRE(0 <= y0 && y0 <= y1 && y1 <= H, "%s: bad row range [%d, %d) of %d", what, y0, y1, H);
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0 && ((uintptr_t)canvas_dev & 15) == 0 && ((uintptr_t)args_dev & 15) == 0,
                 "%s: pitch %lld must be >= 3*W and a multiple of 16, canvas and argument block 16-byte aligned", what, (long long)pitch);
    USDU_REQUIRE(max_ctas >= 1, "%s: max_ctas must be >= 1, got %d", what, max_ctas);
    return USDU_OK;
}

int usdu_quantize_rows_streamed(const usdu_stream_args* args_dev, uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                                int y0, int y1, int max_ctas, void* stream) {
    const int s = check_streamed("usdu_quantize_rows_streamed", args_dev, canvas_dev, B, H, W, pitch, y0, y1, max_ctas);
    if (s != USDU_OK || y1 == y0) return s;
    const int W3 = W * 3;
    const int64_t blocks = ((int64_t)B * (y1 - y0) * ((W3 + 15) / 16) + kThreads - 1) / kThreads;
    const int grid = (int)(blocks < max_ctas ? blocks : max_ctas);
    quantize_rows_streamed_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(args_dev, canvas_dev, B * (y1 - y0), W3, pitch, H, y0, y1 - y0);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_dequantize_rows_streamed(const uint8_t* canvas_dev, const usdu_stream_args* args_dev, int B, int H, int W,
                                  int64_t pitch, int y0, int y1, int max_ctas, void* stream) {
    const int s = check_streamed("usdu_dequantize_rows_streamed", args_dev, canvas_dev, B, H, W, pitch, y0, y1, max_ctas);
    if (s != USDU_OK || y1 == y0) return s;
    const int W3 = W * 3;
    int gx = (W3 / 4 + kThreads * 4 - 1) / (kThreads * 4);          // ~4 words per thread along a row, as usdu_dequantize_rows
    if (gx > max_ctas) gx = max_ctas;
    int64_t gy = max_ctas / gx;
    const int64_t rows = (int64_t)B * (y1 - y0);
    if (gy > rows) gy = rows;
    if (gy > 65535) gy = 65535;
    dequantize_rows_streamed_kernel<<<dim3(gx, (unsigned)gy), kThreads, 0, (cudaStream_t)stream>>>(canvas_dev, args_dev, (int)rows, W3,
                                                                                                    pitch, H, y0, y1 - y0);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_graph_instantiate(void* graph, int high_priority, void** exec_out) {
    USDU_REQUIRE(graph && exec_out, "usdu_graph_instantiate: null pointer");
    cudaGraph_t g = (cudaGraph_t)graph;
    if (high_priority) {
        int least = 0, greatest = 0;
        USDU_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        size_t n = 0;
        USDU_CUDA(cudaGraphGetNodes(g, nullptr, &n));
        cudaGraphNode_t* nodes = (cudaGraphNode_t*)malloc((n ? n : 1) * sizeof(cudaGraphNode_t));
        USDU_REQUIRE(nodes != nullptr, "usdu_graph_instantiate: out of host memory");
        cudaError_t e = cudaGraphGetNodes(g, nodes, &n);
        for (size_t i = 0; e == cudaSuccess && i < n; ++i) {
            cudaGraphNodeType type;
            e = cudaGraphNodeGetType(nodes[i], &type);
            if (e != cudaSuccess || type != cudaGraphNodeTypeKernel) continue;
            cudaKernelNodeParams p = {};
            // a node the runtime cannot describe (a driver-API launch) is not one of the streamed casts
            if (cudaGraphKernelNodeGetParams(nodes[i], &p) != cudaSuccess) {
                (void)cudaGetLastError();
                p.func = nullptr;
            }
            if (p.func == (void*)quantize_rows_streamed_kernel || p.func == (void*)dequantize_rows_streamed_kernel) continue;
            cudaLaunchAttributeValue v = {};
            v.priority = greatest;
            e = cudaGraphKernelNodeSetAttribute(nodes[i], cudaLaunchAttributePriority, &v);
        }
        free(nodes);
        USDU_CUDA(e);
    }
    cudaGraphExec_t exec = nullptr;
    USDU_CUDA(cudaGraphInstantiateWithFlags(&exec, g, high_priority ? cudaGraphInstantiateFlagUseNodePriority : 0));
    *exec_out = (void*)exec;
    return USDU_OK;
}

int usdu_graph_launch(void* exec, void* stream) {
    USDU_REQUIRE(exec, "usdu_graph_launch: null graph");
    USDU_CUDA(cudaGraphLaunch((cudaGraphExec_t)exec, (cudaStream_t)stream));
    return USDU_OK;
}

int usdu_graph_exec_destroy(void* exec) {
    if (exec) USDU_CUDA(cudaGraphExecDestroy((cudaGraphExec_t)exec));
    return USDU_OK;
}

int usdu_gather_dequantize(const uint8_t* const* slab_canvas_dev, const int32_t* slab_rows, int n_slabs, float* img_dev,
                           int B, int H, int W, int64_t pitch, void* stream) {
    USDU_REQUIRE(slab_canvas_dev && slab_rows && img_dev, "usdu_gather_dequantize: null pointer");
    USDU_REQUIRE(n_slabs >= 1 && n_slabs <= USDU_MAX_SLABS, "usdu_gather_dequantize: 1..%d slabs, got %d", USDU_MAX_SLABS, n_slabs);
    USDU_REQUIRE(B > 0 && H > 0 && W > 0, "usdu_gather_dequantize: bad shape %dx%dx%d", B, H, W);
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0, "usdu_gather_dequantize: pitch %lld must be >= 3*W and a multiple of 16", (long long)pitch);
    USDU_REQUIRE(slab_rows[0] == 0 && slab_rows[n_slabs] == H, "usdu_gather_dequantize: the slabs must tile rows 0..%d", H);
    const int W3 = W * 3;
    bool vec = (W3 % 4 == 0) && (((uintptr_t)img_dev & 15) == 0);
    GatherArgs a;
    a.n = n_slabs;
    for (int q = 0; q < n_slabs; ++q) {
        USDU_REQUIRE(slab_canvas_dev[q] != nullptr && slab_rows[q] <= slab_rows[q + 1], "usdu_gather_dequantize: bad slab %d", q);
        a.base[q] = slab_canvas_dev[q];
        a.y[q] = slab_rows[q];
        vec = vec && (((uintptr_t)slab_canvas_dev[q] & 15) == 0);
    }
    a.y[n_slabs] = H;
    if (!vec) {                                   // odd widths: slab by slab through the scalar path
        for (int q = 0; q < n_slabs; ++q) {
            int s = usdu_dequantize_rows(slab_canvas_dev[q], img_dev, B, H, W, pitch, slab_rows[q], slab_rows[q + 1], stream);
            if (s != USDU_OK) return s;
        }
        return USDU_OK;
    }
    const int gx = (W3 + kThreads * 16 - 1) / (kThreads * 16);
    int64_t gy = (int64_t)B * H;
    if (gy > 65535) gy = 65535;
    gather_dequantize_kernel<<<dim3(gx, (unsigned)gy), kThreads, 0, (cudaStream_t)stream>>>(a, img_dev, B * H, H, W3, pitch);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_gather_canvas(const uint8_t* const* slab_canvas_dev, const int32_t* slab_rows, int n_slabs, uint8_t* canvas_dev,
                       int B, int H, int W, int64_t pitch, void* stream) {
    USDU_REQUIRE(slab_canvas_dev && slab_rows && canvas_dev, "usdu_gather_canvas: null pointer");
    USDU_REQUIRE(n_slabs >= 1 && n_slabs <= USDU_MAX_SLABS, "usdu_gather_canvas: 1..%d slabs, got %d", USDU_MAX_SLABS, n_slabs);
    USDU_REQUIRE(B > 0 && H > 0 && W > 0, "usdu_gather_canvas: bad shape %dx%dx%d", B, H, W);
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0 && ((uintptr_t)canvas_dev & 15) == 0, "usdu_gather_canvas: pitch / base must be multiples of 16");
    USDU_REQUIRE(slab_rows[0] == 0 && slab_rows[n_slabs] == H, "usdu_gather_canvas: the slabs must tile rows 0..%d", H);
    GatherArgs a;
    a.n = n_slabs;
    for (int q = 0; q < n_slabs; ++q) {
        USDU_REQUIRE(slab_canvas_dev[q] != nullptr && ((uintptr_t)slab_canvas_dev[q] & 15) == 0 && slab_rows[q] <= slab_rows[q + 1],
                     "usdu_gather_canvas: bad slab %d", q);
        a.base[q] = slab_canvas_dev[q];
        a.y[q] = slab_rows[q];
    }
    a.y[n_slabs] = H;
    const int row_bytes = (W * 3 + 15) / 16 * 16;                // whole 16-byte words of a row (<= pitch)
    const int gx = (row_bytes / 16 + kThreads - 1) / kThreads;
    int64_t gy = (int64_t)B * H;
    if (gy > 65535) gy = 65535;
    gather_canvas_kernel<<<dim3(gx, (unsigned)gy), kThreads, 0, (cudaStream_t)stream>>>(a, canvas_dev, B * H, H, row_bytes, pitch);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_dequantize_canvas(const uint8_t* canvas_dev, float* img_dev, int B, int H, int W, int64_t pitch,
                           void* stream) {
    USDU_REQUIRE(H > 0, "usdu_dequantize_canvas: bad shape %dx%dx%d", B, H, W);
    return usdu_dequantize_rows(canvas_dev, img_dev, B, H, W, pitch, 0, H, stream);
}

int usdu_pack_tiles_u8(const float* src_dev, uint8_t* dst_dev, int64_t n, void* stream) {
    USDU_REQUIRE(n >= 0, "usdu_pack_tiles_u8: negative count");
    if (n == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && dst_dev, "usdu_pack_tiles_u8: null pointer");
    USDU_REQUIRE((((uintptr_t)src_dev | (uintptr_t)dst_dev) & 15) == 0, "usdu_pack_tiles_u8: pointers must be 16-byte aligned");
    if (n == 0) return USDU_OK;
    const int grid = grid_for(((n >> 4) + kThreads) / kThreads);
    pack_u8_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(src_dev, dst_dev, n);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_unpack_tiles_f32(const uint8_t* src_dev, float* dst_dev, int64_t n, void* stream) {
    USDU_REQUIRE(n >= 0, "usdu_unpack_tiles_f32: negative count");
    if (n == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && dst_dev, "usdu_unpack_tiles_f32: null pointer");
    USDU_REQUIRE((((uintptr_t)src_dev | (uintptr_t)dst_dev) & 15) == 0, "usdu_unpack_tiles_f32: pointers must be 16-byte aligned");
    if (n == 0) return USDU_OK;
    const int grid = grid_for(((n >> 4) + kThreads) / kThreads);
    unpack_f32_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(src_dev, dst_dev, n);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_t0_denoise(const float* tiles_dev, const float* noise_scaled_dev, float* out_dev, int64_t n, int64_t frame,
                    float one_minus_d, void* stream) {
    USDU_REQUIRE(n >= 0 && frame > 0, "usdu_t0_denoise: bad sizes");
    if (n == 0) return USDU_OK;
    USDU_REQUIRE(tiles_dev && noise_scaled_dev && out_dev, "usdu_t0_denoise: null pointer");
    USDU_REQUIRE(n % 4 == 0 && frame % 4 == 0 && n % frame == 0, "usdu_t0_denoise: n and frame must be multiples of 4, n of frame");
    USDU_REQUIRE((((uintptr_t)tiles_dev | (uintptr_t)noise_scaled_dev | (uintptr_t)out_dev) & 15) == 0, "usdu_t0_denoise: pointers must be 16-byte aligned");
    const int grid = grid_for((n / 4 + kThreads - 1) / kThreads);
    USDU_CUDA(launch_pdl(t0_denoise_kernel, dim3(grid), dim3(kThreads), 0, (cudaStream_t)stream,
                         reinterpret_cast<const float4*>(tiles_dev), reinterpret_cast<const float4*>(noise_scaled_dev),
                         reinterpret_cast<float4*>(out_dev), n / 4, frame / 4, one_minus_d));
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

static int mask_ext_len(const int32_t* s, int rad, bool horiz) {
    const int n_canvas = horiz ? s[0] : s[1];
    const int w0 = horiz ? s[6] : s[7], w1 = horiz ? s[8] : s[9];
    const int ext = 3 * (rad + 1);
    return min(n_canvas, w1 + ext) - max(0, w0 - ext);
}

int64_t usdu_mask_scratch_bytes(const int32_t* specs_host, int n_specs) {
    if (!specs_host || n_specs < 0) {
        set_error("usdu_mask_scratch_bytes: bad arguments");
        return USDU_ERR_INVALID;
    }
    int64_t total = (int64_t)n_specs * sizeof(MaskSpecDev) + 256;
    for (int i = 0; i < n_specs; ++i) {
        const int32_t* s = specs_host + (int64_t)i * USDU_MASK_WORDS;
        const int64_t ew = s[8] - s[6], eh = s[9] - s[7];
        total += ew + 256 * eh;
    }
    return total;
}

int usdu_build_feather_masks(const int32_t* specs_host, int n_specs, uint8_t* mask_pool_dev,
                             uint8_t* scratch_dev, void* stream) {
    USDU_REQUIRE(specs_host && mask_pool_dev && scratch_dev, "usdu_build_feather_masks: null pointer");
    USDU_REQUIRE(n_specs > 0, "usdu_build_feather_masks: n_specs must be > 0");
    MaskSpecDev* host = new MaskSpecDev[n_specs];
    int64_t off = ((int64_t)n_specs * sizeof(MaskSpecDev) + 255) / 256 * 256;
    int max_len = 1;
    for (int i = 0; i < n_specs; ++i) {
        const int32_t* s = specs_host + (int64_t)i * USDU_MASK_WORDS;
        MaskSpecDev& d = host[i];
        d.W = s[0]; d.H = s[1]; d.bx1 = s[2]; d.by1 = s[3]; d.bx2 = s[4]; d.by2 = s[5];
        d.x1 = s[6]; d.y1 = s[7]; d.x2 = s[8]; d.y2 = s[9];
        d.blur = s[10]; d.out_off = (int64_t)(uint32_t)s[11]; d.out_pitch = s[12];
        bool ok = d.W > 0 && d.H > 0 && d.x1 >= 0 && d.y1 >= 0 && d.x2 > d.x1 && d.y2 > d.y1 && d.x2 <= d.W &&
                  d.y2 <= d.H && d.out_pitch >= d.x2 - d.x1 && d.blur >= 0;
        if (!ok) {
            delete[] host;
            set_error("usdu_build_feather_masks: spec %d is inconsistent", i);
            return USDU_ERR_INVALID;
        }
        d.rad = -1; d.ww = 0; d.fw = 0;
        if (d.blur > 0) {
            int32_t rad;
            int st = usdu_box_blur_params((float)d.blur, &rad, &d.ww, &d.fw);
            if (st != USDU_OK) { delete[] host; return st; }
            d.rad = rad;
        }
        d.scratch_off = off;
        off += (int64_t)(d.x2 - d.x1) + 256LL * (d.y2 - d.y1);
        max_len = max(max_len, max(mask_ext_len(s, d.rad, true), mask_ext_len(s, d.rad, false)));
    }
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemcpyAsync(scratch_dev, host, (size_t)n_specs * sizeof(MaskSpecDev), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // `host` is pageable and freed below
    delete[] host;
    USDU_CUDA(e);
    const size_t smem = 2 * (size_t)((max_len + 15) / 16 * 16);
    int s2 = smem_optin((const void*)mask_profiles_kernel, smem);
    if (s2 != USDU_OK) return s2;
    const MaskSpecDev* specs_dev = reinterpret_cast<const MaskSpecDev*>(scratch_dev);
    mask_profiles_kernel<<<dim3(257, n_specs), kThreads, smem, st>>>(specs_dev, scratch_dev, (int)(smem / 2));
    USDU_CUDA(cudaGetLastError());
    mask_expand_kernel<<<dim3(64, n_specs), kThreads, 0, st>>>(specs_dev, scratch_dev, mask_pool_dev);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_tile_crop_resize(const uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                          const int32_t* tiles_dev, const int32_t* tabs_dev, const int32_t* items_dev,
                          int n_items, int patch_w, int patch_h, float* out_dev, int flags, void* stream) {
    USDU_REQUIRE(canvas_dev && tiles_dev && items_dev && out_dev, "usdu_tile_crop_resize: null pointer");
    USDU_REQUIRE(B > 0 && H > 0 && W > 0 && n_items >= 0, "usdu_tile_crop_resize: bad shape");
    USDU_REQUIRE(B <= 65535, "usdu_tile_crop_resize: batch %d exceeds grid.y limit", B);
    USDU_REQUIRE(patch_w > 0 && patch_h > 0, "usdu_tile_crop_resize: patch capacity must be positive");
    if (n_items == 0) return USDU_OK;
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0, "usdu_tile_crop_resize: pitch must be >= 3*W and a multiple of 16");
    if (flags & USDU_FLAG_MMA) {
        USDU_REQUIRE(tabs_dev != nullptr, "usdu_tile_crop_resize: tensor-core path needs tables");
        return mma::launch_crop(canvas_dev, 0, B, H, W, pitch, tabs_dev, items_dev, n_items, patch_w, patch_h, out_dev,
                                (flags & USDU_FLAG_MMA_KS2) ? 1 : 0, (cudaStream_t)stream);
    }
    if (flags & USDU_FLAG_FAST) {
        USDU_REQUIRE(tabs_dev != nullptr, "usdu_tile_crop_resize: fast path needs tables");
        return fast::launch_crop(canvas_dev, B, H, W, pitch, tiles_dev, tabs_dev, items_dev, n_items, patch_w, patch_h,
                                 out_dev, (cudaStream_t)stream);
    }
    const int in_pitch = (patch_w * 3 + 15) / 16 * 16;
    const size_t smem = (size_t)patch_h * in_pitch + (size_t)patch_h * BW * 3;
    int s = smem_optin((const void*)crop_resize_kernel, smem);
    if (s != USDU_OK) return s;
    int blk_h = (flags >> 8) & 0xFF, blk_w = (flags >> 16) & 0xFF;     // generic path: optional smaller blocks
    if (blk_h <= 0 || blk_h > BH) blk_h = BH;
    if (blk_w <= 0 || blk_w > BW) blk_w = BW;
    crop_resize_kernel<<<dim3(n_items, B), kThreads, smem, (cudaStream_t)stream>>>(
        canvas_dev, H, W, pitch, tiles_dev, tabs_dev, items_dev, out_dev, in_pitch, patch_h, blk_w, blk_h);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_tile_crop_resize_f32(const float* image_dev, int B, int H, int W, const int32_t* tabs_dev, const int32_t* items_dev,
                              int n_items, int patch_w, int patch_h, float* out_dev, int flags, void* stream) {
    USDU_REQUIRE(image_dev && tabs_dev && items_dev && out_dev, "usdu_tile_crop_resize_f32: null pointer");
    USDU_REQUIRE(B > 0 && H > 0 && W > 0 && n_items >= 0, "usdu_tile_crop_resize_f32: bad shape");
    USDU_REQUIRE(B <= 65535, "usdu_tile_crop_resize_f32: batch %d exceeds grid.y limit", B);
    USDU_REQUIRE(flags & USDU_FLAG_MMA, "usdu_tile_crop_resize_f32: tensor-core job records only (USDU_FLAG_MMA)");
    if (n_items == 0) return USDU_OK;
    return mma::launch_crop(image_dev, 1, B, H, W, (int64_t)W * 3, tabs_dev, items_dev, n_items, patch_w, patch_h, out_dev,
                            (flags & USDU_FLAG_MMA_KS2) ? 1 : 0, (cudaStream_t)stream);
}

int usdu_tile_blend(uint8_t* canvas_dev, int B, int H, int W, int64_t pitch, const int32_t* tiles_dev,
                    const int32_t* tabs_dev, const uint8_t* mask_pool_dev, const int32_t* items_dev,
                    int n_items, const int32_t* cover_dev, int patch_w, int patch_h, const void* src_dev,
                    int src_is_u8, int flags, void* stream) {
    USDU_REQUIRE(canvas_dev && tiles_dev && mask_pool_dev && items_dev && src_dev && (cover_dev || (flags & (USDU_FLAG_FAST | USDU_FLAG_MMA))),
                 "usdu_tile_blend: null pointer");
    USDU_REQUIRE(B > 0 && H > 0 && W > 0 && n_items >= 0, "usdu_tile_blend: bad shape");
    USDU_REQUIRE(B <= 65535, "usdu_tile_blend: batch %d exceeds grid.y limit", B);
    USDU_REQUIRE(patch_w > 0 && patch_h > 0, "usdu_tile_blend: patch capacity must be positive");
    if (n_items == 0) return USDU_OK;
    USDU_REQUIRE(pitch >= 3LL * W && pitch % 16 == 0, "usdu_tile_blend: pitch must be >= 3*W and a multiple of 16");
    if (flags & USDU_FLAG_MMA) {
        USDU_REQUIRE(tabs_dev != nullptr, "usdu_tile_blend: tensor-core path needs tables");
        USDU_REQUIRE(((uintptr_t)src_dev & 15) == 0, "usdu_tile_blend: src must be 16-byte aligned");
        return mma::launch_blend(canvas_dev, B, H, W, pitch, tabs_dev, mask_pool_dev, items_dev, n_items, patch_w, patch_h, src_dev,
                                 src_is_u8, (flags >> 8) & 0xFF, (flags & USDU_FLAG_MMA_KS2) ? 1 : 0, (cudaStream_t)stream);
    }
    if (flags & USDU_FLAG_FAST) {
        USDU_REQUIRE(tabs_dev != nullptr, "usdu_tile_blend: fast path needs tables");
        USDU_REQUIRE(((uintptr_t)src_dev & 15) == 0, "usdu_tile_blend: src must be 16-byte aligned");
        return fast::launch_blend(canvas_dev, B, H, W, pitch, tiles_dev, tabs_dev, mask_pool_dev, items_dev, n_items,
                                  cover_dev, patch_w, patch_h, src_dev, src_is_u8, (flags >> 8) & 0xFF,
                                  (flags & USDU_FLAG_REMOTE_CANVAS) ? 1 : 0, (cudaStream_t)stream);
    }
    int blk_h = (flags >> 8) & 0xFF, blk_w = (flags >> 16) & 0xFF;     // generic path: optional smaller blocks
    if (blk_h <= 0 || blk_h > BH) blk_h = BH;
    if (blk_w <= 0 || blk_w > BW) blk_w = BW;
    const int in_pitch = (patch_w * 3 + 15) / 16 * 16;
    const size_t head = (size_t)BH * BW * 3 + (size_t)patch_h * blk_w * 3;
    const bool direct = head + (size_t)patch_h * in_pitch > kMaxSmem;  // the patch does not fit: read the tile itself
    const size_t smem = direct ? head : head + (size_t)patch_h * in_pitch;
    void (*fn)(uint8_t*, int, int, int64_t, const int32_t*, const int32_t*, const uint8_t*, const int32_t*, const int32_t*,
               const void*, int, int, int, int) =
        src_is_u8 ? (direct ? blend_kernel<true, true> : blend_kernel<true, false>)
                  : (direct ? blend_kernel<false, true> : blend_kernel<false, false>);
    int s = smem_optin((const void*)fn, smem);
    if (s != USDU_OK) return s;
    fn<<<dim3(n_items, B), kThreads, smem, (cudaStream_t)stream>>>(
        canvas_dev, H, W, pitch, tiles_dev, tabs_dev, mask_pool_dev, items_dev, cover_dev, src_dev, in_pitch, patch_h, blk_w, blk_h);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

}  // extern "C"
