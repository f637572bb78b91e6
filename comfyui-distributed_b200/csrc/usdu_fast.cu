// usdu_fast.cu -- fast crop+LANCZOS and LANCZOS-back+composite kernels (sm_90a).
// See usdu_fast.cuh for the engine; this file holds staging, epilogues and launchers.
#include "usdu_fast.cuh"
#include "usdu_tma.cuh"
#include <string.h>
#include <stdlib.h>

namespace usdu {
namespace fast {

// Transpose 4 registers (rows) x 4 bytes (columns) -> 4 words, word j = byte j of rows 0..3.
__device__ __forceinline__ void transpose4x4(uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t (&o)[4]) {
    const uint32_t a = __byte_perm(r0, r1, 0x5140), b = __byte_perm(r0, r1, 0x7362);   // (r0.b0 r1.b0 r0.b1 r1.b1), (.. b2 b3)
    const uint32_t c = __byte_perm(r2, r3, 0x5140), d = __byte_perm(r2, r3, 0x7362);
    o[0] = __byte_perm(a, c, 0x5410);
    o[1] = __byte_perm(a, c, 0x7632);
    o[2] = __byte_perm(b, d, 0x5410);
    o[3] = __byte_perm(b, d, 0x7632);
}

// ---- staging: u8 pixel-interleaved rows -> planar row-packed words ---------------------------
// src(r, byte) = row r (0..rows) of the patch, `bytes_avail` valid bytes per row starting at the
// 4-byte aligned address src + r * pitch.  Byte b of a row is channel (b + phase) % 3 of pixel
// (b + phase) / 3 - px_shift ... the caller arranges src so that byte 0 is channel 0 of patch
// pixel -lead (lead in 0..3 pixels, i.e. src points 3*lead bytes before the patch start and is
// 4-byte aligned).  Rows >= rows_valid are clamped to the last valid row.
__device__ __forceinline__ void stage_u8(uint32_t* __restrict__ in, int xw, const uint8_t* __restrict__ src,
                                         int64_t pitch, int rows, int rows_valid, int px_count, int lead) {
    // unit = (group g of 4 rows, chunk of 4 pixels = 12 bytes = 3 aligned words)
    const int chunks = (px_count + lead + 3) >> 2;
    const int groups = (rows + 3) >> 2;
    for (int i = threadIdx.x; i < groups * chunks; i += kT) {
        const int g = i / chunks, ch = i - g * chunks;
        uint32_t w[4][3];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int rr = min(4 * g + r, rows_valid - 1);
            const uint32_t* p = reinterpret_cast<const uint32_t*>(src + (int64_t)rr * pitch) + ch * 3;
            w[r][0] = __ldg(p);
            w[r][1] = __ldg(p + 1);
            w[r][2] = __ldg(p + 2);
        }
        // 12 byte columns: col j -> pixel ch*4 + j/3 - lead, channel j%3
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            uint32_t t[4];
            transpose4x4(w[0][k], w[1][k], w[2][k], w[3][k], t);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = k * 4 + j;              // compile time
                const int px = ch * 4 + col / 3 - lead;
                const int c = col % 3;
                if (px >= 0 && px < xw) in[(size_t)(g * 3 + c) * xw + px] = t[j];
            }
        }
    }
}

// fp32 source in [0,1] -> quantise (Q1) -> planar row-packed.  src points at the first float of
// a 12-float (4 pixel) aligned chunk that contains the patch start; lead = pixels before it.  Evict-first loads: the
// source is dead once blended (see usdu_mma.cu stage_f32).
__device__ __forceinline__ void stage_f32(uint32_t* __restrict__ in, int xw, const float* __restrict__ src,
                                          int64_t pitch_f, int rows, int rows_valid, int px_count, int lead) {
    const int chunks = (px_count + lead + 3) >> 2;
    const int groups = (rows + 3) >> 2;
    for (int i = threadIdx.x; i < groups * chunks; i += kT) {
        const int g = i / chunks, ch = i - g * chunks;
        uint32_t q[4][3];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int rr = min(4 * g + r, rows_valid - 1);
            const float4* p = reinterpret_cast<const float4*>(src + (int64_t)rr * pitch_f) + ch * 3;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float4 f = __ldcs(p + k);
                q[r][k] = quant_u8(f.x) | (quant_u8(f.y) << 8) | (quant_u8(f.z) << 16) | (quant_u8(f.w) << 24);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            uint32_t t[4];
            transpose4x4(q[0][k], q[1][k], q[2][k], q[3][k], t);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = k * 4 + j;
                const int px = ch * 4 + col / 3 - lead;
                const int c = col % 3;
                if (px >= 0 && px < xw) in[(size_t)(g * 3 + c) * xw + px] = t[j];
            }
        }
    }
}

// TMA path of the crop kernel: the canvas patch arrives row-major in shared memory as two
// boxes of kBoxB bytes x kBoxR rows (one bulk-tensor load each); this pass re-lays it out planar
// and row-packed.  Same unit decomposition as stage_u8, LDS instead of LDG.
constexpr int kBoxB = 256;   // bytes per box row (TMA maximum); 2 boxes cover 15 + 3*(patch_w + 3) bytes
constexpr int kBoxR = 40;
// `lead_b` = bytes between the 16-byte aligned box start (a TMA requirement on the inner
// coordinate, measured: tools/ubench/tma_probe.cu) and the first staged pixel.
__device__ __forceinline__ void stage_from_raw(uint32_t* __restrict__ in, int xw, const uint8_t* __restrict__ raw,
                                               int rows, int px_count, int lead, int lead_b) {
    const int chunks = (px_count + lead + 3) >> 2;
    const int groups = (rows + 3) >> 2;
    for (int i = threadIdx.x; i < groups * chunks; i += kT) {
        const int g = i / chunks, ch = i - g * chunks;
        uint32_t w[4][3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int o = lead_b + 12 * ch + 4 * k;                       // byte offset in the virtual 512-byte row
            const uint8_t* base = raw + (size_t)(o >> 8) * (kBoxR * kBoxB) + (o & 255);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int rr = min(4 * g + r, rows - 1);
                w[r][k] = *reinterpret_cast<const uint32_t*>(base + rr * kBoxB);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            uint32_t t[4];
            transpose4x4(w[0][k], w[1][k], w[2][k], w[3][k], t);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = k * 4 + j;
                const int px = ch * 4 + col / 3 - lead;
                const int c = col % 3;
                if (px >= 0 && px < xw) in[(size_t)(g * 3 + c) * xw + px] = t[j];
            }
        }
    }
}

// Load the job record of this CTA (thread 0..7 -> one int4 each) and the V-axis rows.
__device__ __forceinline__ void load_job(int32_t* job_sm, const int32_t* __restrict__ jobs, int idx) {
    if (threadIdx.x < USDU_JOB_WORDS / 4)
        reinterpret_cast<int4*>(job_sm)[threadIdx.x] =
            __ldg(reinterpret_cast<const int4*>(jobs + (size_t)idx * USDU_JOB_WORDS) + threadIdx.x);
}

__device__ __forceinline__ void stage_rows_v(int32_t* rows_sm, const int32_t* __restrict__ tabs, const JobView& J) {
    const int q = J[USDU_J_TAPS_V] <= USDU_FAST_TAPS ? 2 : 4;        // int4 per packed row (8 or 16 int32)
    for (int i = threadIdx.x; i < FBH * q; i += kT) {
        const int r = i / q, part = i - r * q;
        const int o = clampi(J[USDU_J_OY_BASE] + r, 0, J[USDU_J_N_OUT_V] - 1);
        reinterpret_cast<int4*>(rows_sm)[i] =
            __ldg(reinterpret_cast<const int4*>(tabs + J[USDU_J_ROWS_V] + (size_t)o * (4 * q)) + part);
    }
}

template <int TAPS>
__device__ __forceinline__ PackedRow<TAPS> load_row_h(const int32_t* __restrict__ tabs, const JobView& J) {
    const int o = clampi(J[USDU_J_OX_BASE] + (int)(threadIdx.x % FBW), 0, J[USDU_J_N_OUT_H] - 1);
    const int4* p = reinterpret_cast<const int4*>(tabs + J[USDU_J_ROWS_H] + (size_t)o * (TAPS + 1));
    return read_row<TAPS>([&](int i) { return __ldg(p + i); });
}

constexpr int kUpTaps = 6;   // taps of an up-scaling (or size-keeping) LANCZOS axis: blend of every uniform tile

// stage -> (sync) -> H pass for one job; the tap count of the axis picks the instantiation
template <class Stage>
__device__ __forceinline__ void stage_and_hpass(const int32_t* __restrict__ tabs, const JobView& J, uint32_t* in, uint8_t* mid,
                                                int xw, Stage stage) {
    if (J[USDU_J_TAPS_H] <= USDU_FAST_TAPS) {
        const PackedRow<USDU_FAST_TAPS> rh = load_row_h<USDU_FAST_TAPS>(tabs, J);    // in flight during staging
        stage();
        __syncthreads();
        if (J[USDU_J_TAPS_H] <= kUpTaps)
            hpass<USDU_FAST_TAPS, kUpTaps>(in, mid, rh, J[USDU_J_IX0], J[USDU_J_ROWS], xw);
        else
            hpass<USDU_FAST_TAPS>(in, mid, rh, J[USDU_J_IX0], J[USDU_J_ROWS], xw);
    } else {
        const PackedRow<MAXTAPS> rh = load_row_h<MAXTAPS>(tabs, J);
        stage();
        __syncthreads();
        hpass<MAXTAPS>(in, mid, rh, J[USDU_J_IX0], J[USDU_J_ROWS], xw);
    }
}

template <class Epilogue>
__device__ __forceinline__ void vpass_any(const uint8_t* mid, const int32_t* rows_v, const JobView& J, Epilogue& epi, int r0, int r1) {
    if (J[USDU_J_TAPS_V] <= kUpTaps)
        vpass<USDU_FAST_TAPS, kUpTaps>(mid, rows_v, J[USDU_J_IY0], epi, r0, r1);
    else if (J[USDU_J_TAPS_V] <= USDU_FAST_TAPS)
        vpass<USDU_FAST_TAPS, USDU_FAST_TAPS>(mid, rows_v, J[USDU_J_IY0], epi, r0, r1);
    else
        vpass<MAXTAPS, MAXTAPS>(mid, rows_v, J[USDU_J_IY0], epi, r0, r1);
}

// ======================================================================================
// crop + resize
// ======================================================================================
struct CropEpilogue {
    float* dst;          // &out[tile][b][oy0][ox0][0]
    int64_t row_pitch;   // floats per output row
    int ow3;
    const float* lut;
    struct Pre {};
    __device__ __forceinline__ Pre prefetch(int, int) const { return Pre{}; }
    __device__ __forceinline__ void row(const Pre&, int r, int strip, const uint32_t (&s)[4]) {
        if (4 * strip < ow3) {   // ow3 is a multiple of 4 (pw % 8 == 0)
            float4 o;
            o.x = lut[s[0]]; o.y = lut[s[1]]; o.z = lut[s[2]]; o.w = lut[s[3]];
            store_handoff(dst + (int64_t)r * row_pitch + 4 * strip, o);
        }
    }
};

// kTma: stage the canvas patch with two cp.async.bulk.tensor.2d loads (UTMALDG) instead of LDG.
template <bool kTma>
__global__ void __launch_bounds__(kT, 4)
crop_fast_kernel(const uint8_t* __restrict__ canvas, int H, int64_t pitch, const int32_t* __restrict__ tabs,
                 const int32_t* __restrict__ jobs, float* __restrict__ out, int patch_w, int patch_h, int W3,
                 const __grid_constant__ CUtensorMap cmap) {
    extern __shared__ __align__(128) uint8_t smem[];
    // [mid | raw (TMA boxes), aliased: raw is dead before the H pass writes mid] [job, rows_v] [lut] [bar] [in]
    const size_t region = kTma ? max(mid_bytes(patch_h), (size_t)2 * kBoxR * kBoxB) : mid_bytes(patch_h);
    uint8_t* mid = smem;
    uint8_t* raw = smem;
    int32_t* job_sm = reinterpret_cast<int32_t*>(smem + region);
    int32_t* rows_v = job_sm + USDU_JOB_WORDS;
    float* lut = reinterpret_cast<float*>(smem + region + kHeadBytes);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + region + kHeadBytes + 1024);
    uint32_t* in = reinterpret_cast<uint32_t*>(smem + region + kHeadBytes + 1024 + 16);
    pdl_launch_dependents();
    load_job(job_sm, jobs, blockIdx.x);
    if (kTma && threadIdx.x == 0) tma::mbar_init(bar, 1);
    for (int i = threadIdx.x; i < 256; i += kT) lut[i] = dequant_u8_fast(i);
    __syncthreads();
    const JobView J{job_sm};
    const int b = blockIdx.y;
    const int xw = plane_words(patch_w);
    stage_rows_v(rows_v, tabs, J);
    pdl_wait();                                // the canvas is the previous kernel's output
    if (kTma && threadIdx.x == 0) {
        const int x = (J[USDU_J_SRC_A] * 3) & ~15, y = J[USDU_J_SRC_B];           // 16-byte aligned box start
        // second box only when the patch needs it and it starts inside the canvas row
        const bool two = (J[USDU_J_SRC_A] * 3 - x) + (J[USDU_J_COLS] + J[USDU_J_LEAD]) * 3 > kBoxB && x + kBoxB < W3;
        tma::mbar_expect_tx(bar, (two ? 2 : 1) * kBoxR * kBoxB);
        tma::load_3d(raw, &cmap, x, y, b, bar);
        if (two) tma::load_3d(raw + kBoxR * kBoxB, &cmap, x + kBoxB, y, b, bar);
    }
    stage_and_hpass(tabs, J, in, mid, xw, [&]() {
        if (kTma) {
            tma::mbar_wait(bar, 0);
            stage_from_raw(in, xw, raw, J[USDU_J_ROWS], J[USDU_J_COLS], J[USDU_J_LEAD], (J[USDU_J_SRC_A] * 3) & 15);
            // raw is aliased with mid: stage_and_hpass() synchronises before the H pass overwrites it
        } else {
            const uint8_t* src = canvas + ((int64_t)b * H + J[USDU_J_SRC_B]) * pitch + (int64_t)J[USDU_J_SRC_A] * 3;
            stage_u8(in, xw, src, pitch, J[USDU_J_ROWS], J[USDU_J_ROWS], J[USDU_J_COLS], J[USDU_J_LEAD]);
        }
    });
    __syncthreads();
    CropEpilogue epi;
    epi.row_pitch = J[USDU_J_PITCH];
    epi.dst = out + J.i64(USDU_J_OFF_LO) + (int64_t)b * J.i64(USDU_J_FRAME_LO) + (int64_t)J[USDU_J_DST_Y] * epi.row_pitch +
              (int64_t)J[USDU_J_DST_X] * 3;
    epi.ow3 = J[USDU_J_COLS_OUT] * 3;
    epi.lut = lut;
    vpass_any(mid, rows_v, J, epi, 0, J[USDU_J_ROWS_OUT]);
}

// ======================================================================================
// blend
// ======================================================================================
// The canvas block (128 px x bh rows) lives in shared memory for the whole CTA: it arrives with
// two bulk-tensor loads (UTMALDG, 192-byte wide boxes), every tile of the block composites into
// it, and it leaves with two bulk-tensor stores (UTMASTG).  The canvas is read and written once
// per block regardless of how many tiles overlap there, and the epilogue has no global access
// except the feather template.
constexpr int kDBox = FBW * 3 / 2;          // 192 bytes per box row

struct DTile {
    uint8_t* base;
    int bh;                                  // rows per box
    __device__ __forceinline__ uint32_t* word(int r, int strip) const {
        const int col = 4 * strip;
        const int box = col >= kDBox ? 1 : 0;
        return reinterpret_cast<uint32_t*>(base + (size_t)box * bh * kDBox + r * kDBox + (col - box * kDBox));
    }
};

// interior of a tile (alpha == 255 over the whole block): the canvas block becomes S
struct BlendOpaque {
    DTile d;
    struct Pre {};
    __device__ __forceinline__ Pre prefetch(int, int) const { return Pre{}; }
    __device__ __forceinline__ void row(const Pre&, int r, int strip, const uint32_t (&s)[4]) {
        *d.word(r, strip) = s[0] | (s[1] << 8) | (s[2] << 16) | (s[3] << 24);
    }
};

// general case: per-pixel alpha from the feather template, zero outside the tile's sub-rect
struct BlendFeather {
    DTile d;
    const uint8_t* mask;   // template address of block pixel (0,0) (may point outside; guarded by the rect)
    int mpitch;
    int cx0, cx1;          // sub-rect columns in block pixel coordinates (rows are bounded by the caller)
    struct Pre {
        uint32_t aa, ab;   // alpha of the two pixels the 4 bytes touch
        int split;         // bytes [0, split) belong to the first pixel
    };
    __device__ __forceinline__ Pre prefetch(int r, int strip) const {
        const int col = 4 * strip;
        const int pa = col / 3, pb = (col + 3) / 3;          // pb = pa or pa + 1
        const bool ina = pa >= cx0 && pa < cx1, inb = pb >= cx0 && pb < cx1;
        const uint8_t* mrow = mask + (int64_t)r * mpitch;
        Pre p;
        p.aa = ina ? (uint32_t)__ldg(mrow + pa) : 0u;
        p.ab = inb ? (uint32_t)__ldg(mrow + pb) : 0u;
        p.split = 3 * pb - col;
        return p;
    }
    __device__ __forceinline__ void row(const Pre& p, int r, int strip, const uint32_t (&s)[4]) {
        if ((p.aa | p.ab) == 0u) return;
        uint32_t* w = d.word(r, strip);
        if ((p.aa & p.ab) == 255u) {
            *w = s[0] | (s[1] << 8) | (s[2] << 16) | (s[3] << 24);
            return;
        }
        const uint32_t dv = *w;
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t a = i < p.split ? p.aa : p.ab;
            o |= composite8(s[i], (dv >> (8 * i)) & 0xFF, a) << (8 * i);
        }
        *w = o;
    }
};

template <bool kSrcU8>
__global__ void __launch_bounds__(kT, 4)
blend_fast_kernel(const int32_t* __restrict__ tabs, const uint8_t* __restrict__ mask_pool,
                  const int32_t* __restrict__ jobs, const void* __restrict__ src_v, int W3, int patch_w, int patch_h,
                  int block_rows, int remote, const __grid_constant__ CUtensorMap cmap) {
    extern __shared__ __align__(128) uint8_t smem[];
    // [canvas block: 2 boxes x block_rows x 192] [job, rows_v] [bar] [in] [mid]
    const size_t dbytes = (size_t)2 * block_rows * kDBox;
    int32_t* job_sm = reinterpret_cast<int32_t*>(smem + dbytes);
    int32_t* rows_v = job_sm + USDU_JOB_WORDS;
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + dbytes + kHeadBytes);
    uint32_t* in = reinterpret_cast<uint32_t*>(smem + dbytes + kHeadBytes + 16);
    uint8_t* mid = smem + dbytes + kHeadBytes + 16 + in_bytes(patch_w, patch_h);
    const int b = blockIdx.y;
    const int xw = plane_words(patch_w);
    const JobView J{job_sm};
    DTile D{smem, block_rows};
    int idx = blockIdx.x;
    pdl_launch_dependents();
    load_job(job_sm, jobs, idx);
    if (threadIdx.x == 0) tma::mbar_init(bar, 1);
    __syncthreads();
    stage_rows_v(rows_v, tabs, J);
    pdl_wait();                                // canvas and processed tiles come from earlier kernels
    const int bx3 = J[USDU_J_DST_X] * 3, by = J[USDU_J_DST_Y];
    const bool two = bx3 + kDBox < W3;         // the right half exists (a box may not START past the row end)
    if (threadIdx.x == 0) {                    // canvas block -> shared, asynchronously
        tma::mbar_expect_tx(bar, (uint32_t)(two ? dbytes : dbytes / 2));
        tma::load_3d(smem, &cmap, bx3, by, b, bar);
        if (two) tma::load_3d(smem + (size_t)block_rows * kDBox, &cmap, bx3 + kDBox, by, b, bar);
    }
    bool first = true;
    while (idx >= 0) {
        if (!first) {
            __syncthreads();                   // the previous tile's passes are done with job / rows / in / mid
            load_job(job_sm, jobs, idx);
            __syncthreads();
            stage_rows_v(rows_v, tabs, J);
        }
        const int64_t first_el = J.i64(USDU_J_SRC_A) + (int64_t)b * J.i64(USDU_J_FRAME_LO);
        stage_and_hpass(tabs, J, in, mid, xw, [&]() {
            if (kSrcU8)
                stage_u8(in, xw, static_cast<const uint8_t*>(src_v) + first_el, J[USDU_J_PITCH], J[USDU_J_ROWS], J[USDU_J_ROWS],
                         J[USDU_J_COLS], J[USDU_J_LEAD]);
            else
                stage_f32(in, xw, static_cast<const float*>(src_v) + first_el, J[USDU_J_PITCH], J[USDU_J_ROWS], J[USDU_J_ROWS],
                          J[USDU_J_COLS], J[USDU_J_LEAD]);
        });
        __syncthreads();
        if (first) tma::mbar_wait(bar, 0);     // the canvas block has landed
        if (J[USDU_J_FLAGS] & 1) {
            BlendOpaque epi;
            epi.d = D;
            vpass_any(mid, rows_v, J, epi, 0, J[USDU_J_ROWS_OUT]);
        } else {
            BlendFeather epi;
            epi.d = D;
            epi.mpitch = J[USDU_J_MPITCH];
            epi.mask = mask_pool + J.i64(USDU_J_OFF_LO);
            epi.cx0 = J[USDU_J_CX0]; epi.cx1 = J[USDU_J_CX1];
            vpass_any(mid, rows_v, J, epi, J[USDU_J_CY0], J[USDU_J_CY1]);
        }
        idx = J[USDU_J_NEXT];
        first = false;
    }
    tma::fence_async_smem();                   // generic-proxy writes of the block -> visible to the TMA engine
    __syncthreads();
    if (threadIdx.x == 0) {
        tma::store_3d(&cmap, bx3, by, b, smem);
        if (two) tma::store_3d(&cmap, bx3 + kDBox, by, b, smem + (size_t)block_rows * kDBox);
        tma::store_commit();
        if (remote) {                          // peer canvas: the writes must have landed before the grid can be
            tma::store_wait_all();             // followed by a cross-GPU barrier
            __threadfence_system();
        } else {
            tma::store_wait_read();
        }
    }
}

static size_t crop_smem(int patch_w, int patch_h, bool use_tma) {
    const size_t region = use_tma ? max(mid_bytes(patch_h), (size_t)2 * kBoxR * kBoxB) : mid_bytes(patch_h);
    return region + kHeadBytes + 1024 + 16 + in_bytes(patch_w, patch_h);
}
static size_t blend_smem(int patch_w, int patch_h, int block_rows) {
    return (size_t)2 * block_rows * kDBox + kHeadBytes + 16 + in_bytes(patch_w, patch_h) + mid_bytes(patch_h);
}

static int optin(const void* fn, size_t bytes) {
    if (bytes > 227 * 1024) {
        set_error("fast kernel needs %zu bytes of shared memory (> 227 KB)", bytes);
        return USDU_ERR_UNSUPPORTED;
    }
    return raise_smem_limit(fn, bytes);
}

int launch_crop(const uint8_t* canvas, int B, int H, int W, int64_t pitch, const int32_t* tiles, const int32_t* tabs,
                const int32_t* items, int n_items, int patch_w, int patch_h, float* out, cudaStream_t st) {
    // TMA staging needs the patch to fit two kBoxB x kBoxR boxes (always true for scales <= ~1.2)
    CUtensorMap cmap;
    memset(&cmap, 0, sizeof(cmap));
    bool use_tma = patch_h <= kBoxR && 15 + (patch_w + 3) * 3 <= 2 * kBoxB && ((uintptr_t)canvas & 15) == 0;
    if (use_tma) use_tma = tma::encode_u8_3d(&cmap, canvas, (uint64_t)W * 3, (uint64_t)H, (uint64_t)B, (uint64_t)pitch, kBoxB, kBoxR);
    const size_t smem = crop_smem(patch_w, patch_h, use_tma);
    const void* fn = use_tma ? (const void*)crop_fast_kernel<true> : (const void*)crop_fast_kernel<false>;
    int s = optin(fn, smem);
    if (s != USDU_OK) return s;
    if (use_tma)
        USDU_CUDA(launch_pdl(crop_fast_kernel<true>, dim3(n_items, B), dim3(kT), smem, st, canvas, H, pitch, tabs, items, out, patch_w, patch_h, W * 3, cmap));
    else
        USDU_CUDA(launch_pdl(crop_fast_kernel<false>, dim3(n_items, B), dim3(kT), smem, st, canvas, H, pitch, tabs, items, out, patch_w, patch_h, W * 3, cmap));
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int launch_blend(uint8_t* canvas, int B, int H, int W, int64_t pitch, const int32_t* tiles, const int32_t* tabs,
                 const uint8_t* mask_pool, const int32_t* items, int n_items, const int32_t* cover, int patch_w,
                 int patch_h, const void* src, int src_is_u8, int block_rows, int remote, cudaStream_t st) {
    if (block_rows <= 0 || block_rows > FBH) {
        set_error("usdu_tile_blend: fast path needs the block height (1..%d) in flags bits 8..15, got %d", FBH, block_rows);
        return USDU_ERR_INVALID;
    }
    CUtensorMap cmap;
    memset(&cmap, 0, sizeof(cmap));
    if (((uintptr_t)canvas & 15) != 0 ||
        !tma::encode_u8_3d(&cmap, canvas, (uint64_t)W * 3, (uint64_t)H, (uint64_t)B, (uint64_t)pitch, kDBox, block_rows)) {
        set_error("usdu_tile_blend: cannot build the canvas tensor map (cuTensorMapEncodeTiled)");
        return USDU_ERR_CUDA;
    }
    const size_t smem = blend_smem(patch_w, patch_h, block_rows);
    const void* fn = src_is_u8 ? (const void*)blend_fast_kernel<true> : (const void*)blend_fast_kernel<false>;
    int s = optin(fn, smem);
    if (s != USDU_OK) return s;
    if (src_is_u8)
        USDU_CUDA(launch_pdl(blend_fast_kernel<true>, dim3(n_items, B), dim3(kT), smem, st, tabs, mask_pool, items, src, W * 3, patch_w, patch_h, block_rows, remote, cmap));
    else
        USDU_CUDA(launch_pdl(blend_fast_kernel<false>, dim3(n_items, B), dim3(kT), smem, st, tabs, mask_pool, items, src, W * 3, patch_w, patch_h, block_rows, remote, cmap));
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

}  // namespace fast
}  // namespace usdu
