// usdu_mma.cu -- tensor-core crop+LANCZOS and LANCZOS-back+composite kernels (sm_90a).
//
// Pillow's 8-bit resampling pass is a banded integer contraction, out[o] = clip8((2^21 + sum_k in[k] * coef[o][k]) >> 22)
// with 23-bit signed coefficients.  On the CUDA-core integer pipes a tap costs one PRMT + one IMAD per byte
// (usdu_fast.cuh), so the CUDA-core kernels are ALU-pipe bound, far from the HBM roofline.  Here the taps
// run on the tensor cores: mma.sync.m16n8k32 multiplies u8 pixels by 8-bit LIMBS of the coefficients
// (coef = l2 * 65536 + l1 * 256 + l0; l0, l1 unsigned, l2 signed) with exact s32 accumulation, three IMMAs per
// 16 x 8 x 32 tile, recombined with two shift-adds.  |limb sum| <= 64 * 255 * 255 < 2^23, and the recombined value is
// Pillow's accumulator exactly, so the results stay bit-identical (tools/ubench/imma.cu: probe + throughput).
// Hopper's integer wgmma (s8/u8, m64nNk32) would need the pixel operand in shared memory in its core-matrix layout and a
// warpgroup per 64 output rows; the patches here are 16-row M-tiles of 1 or 2 k-steps, so the warp-level IMMA stays.
//
// Both passes put the COEFFICIENTS in the A operand (16 outputs x 32 inputs, built on the host in fragment order:
// build_mma_frags in usdu_plan.cpp) and the PIXELS in B:
//   H pass  M = 16 output pixels of one channel, N = 8 rows, K = 32 input pixels.  Input staged PLANAR (one byte
//           plane per channel), so a B register is 4 consecutive pixels of a row: one aligned LDS.32.
//   V pass  M = 16 output rows, N = 8 byte columns, K = 32 input rows.  The H pass leaves its u8 results ROW-PACKED,
//           word(kg, col) = rows 4kg..4kg+3 of byte column col, so a B register is again one LDS.32.
// A thread owns 2 x 2 results of a 16 x 8 tile; two N-tiles are run side by side and neighbouring lanes swap halves
// (one SHFL) so that every thread ends with 4 consecutive rows (H) or 4 consecutive bytes (V) to pack into one word.
// Shared-memory pitches (plane rows == 16 mod 32 bytes, row groups == 24 mod 32 words) keep every fragment load and
// every store on 32 distinct banks.
#include "usdu_common.cuh"
#include "usdu_tma.cuh"
#include <string.h>

namespace usdu {
namespace mma {

constexpr int kT = 256;                     // 8 warps
// Resident CTAs per SM the kernels are compiled for.  3 = 80 registers: more registers per thread for the small launches
// of the wave loop (1-8 tiles), where per-thread speed counts.  4 = 64 registers: more warps to hide the staging latency on
// machine-filling crop launches.  The crop launcher picks by grid size.
constexpr int kOccSmall = 3, kOccLarge = 4;
constexpr int kLargeGridPerSM = 8;          // CTAs per SM from which the 4-CTA build of the crop is used
constexpr int BWX = USDU_FAST_BLOCK_W;      // 128-pixel wide blocks
constexpr int MIDP = 440;                   // words per row group of the intermediate: >= 3 * 144 columns, == 24 mod 32
constexpr int kDBox = BWX * 3 / 2;          // canvas block = two bulk-tensor boxes of 192 bytes per row
constexpr int kBoxB = 256, kBoxR = 48;      // crop: raw canvas patch = two boxes of 256 bytes x 48 rows

__host__ __device__ inline int plane_pitch(int patch_w) { return (patch_w + 31) / 32 * 32 + 16; }   // bytes, == 16 mod 32
__host__ __device__ inline size_t planes_bytes(int patch_w, int plane_rows) { return (size_t)3 * plane_rows * plane_pitch(patch_w); }
__host__ __device__ inline size_t mid_bytes(int mid_rows) { return (size_t)(mid_rows / 4) * MIDP * 4; }
constexpr size_t kHeadBytes = USDU_JOB_WORDS * 4;

struct JobView {
    const int32_t* j;
    __device__ __forceinline__ int operator[](int i) const { return j[i]; }
    __device__ __forceinline__ int64_t i64(int lo) const { return (int64_t)(uint32_t)j[lo] | ((int64_t)j[lo + 1] << 32); }
};

__device__ __forceinline__ void load_job(int32_t* job_sm, const int32_t* __restrict__ jobs, int idx) {
    if (threadIdx.x < USDU_JOB_WORDS / 4)
        reinterpret_cast<int4*>(job_sm)[threadIdx.x] = __ldg(reinterpret_cast<const int4*>(jobs + (size_t)idx * USDU_JOB_WORDS) + threadIdx.x);
}

// D = A (16 x 32, coefficients) * B (32 x 8, u8 pixels) + C, s32
__device__ __forceinline__ void mma_uu(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_su(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Pillow's accumulator >> 22 of the recombined limbs (limb 0 starts at the rounding constant 2^21); clip8 happens in pack2
__device__ __forceinline__ int combine(int l0, int l1, int l2) {
    return (l0 + (l1 << 8) + (l2 << 16)) >> kPrecisionBits;
}
// (upper << 16) | clip8(hi) << 8 | clip8(lo): one I2IP (cvt.pack.sat) instead of two clamps, a shift and an OR
__device__ __forceinline__ uint32_t pack2(int lo, int hi, uint32_t upper) {
    uint32_t d;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(hi), "r"(lo), "r"(upper));
    return d;
}

// fragment section of a table (usdu_plan.cpp build_mma_frags): {n_mt, ksteps, 0, 0} then per M-tile {k0, 0, 0, 0, fragments of
// (k-step, limb): 32 lanes x 4 registers}.  Everything is addressed from (section, mt, KS): no dependent load in front of
// the fragment loads.
struct FragTable {
    const int32_t* base;       // tabs + section + 4
    __device__ __forceinline__ FragTable(const int32_t* tabs, int section) : base(tabs + section + 4) {}
    template <int KS>
    __device__ __forceinline__ const int32_t* tile(int mt) const { return base + (size_t)mt * (4 + KS * 384); }
    template <int KS>
    __device__ __forceinline__ int k0(int mt) const { return __ldg(tile<KS>(mt)); }
    template <int KS>
    __device__ __forceinline__ void load(uint32_t (&a)[KS][3][4], int mt, int lane) const {
        const int4* f = reinterpret_cast<const int4*>(tile<KS>(mt) + 4);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
            for (int l = 0; l < 3; ++l) {
                const int4 q = __ldg(f + (ks * 3 + l) * 32 + lane);
                a[ks][l][0] = q.x; a[ks][l][1] = q.y; a[ks][l][2] = q.z; a[ks][l][3] = q.w;
            }
    }
};

// Two N-tiles (A: n = 0..7, B: n = 8..15) of one M-tile -> per row half h (m = g, g + 8) one word of 4 consecutive
// n.  Lane t holds n = 2t, 2t+1 of both tiles; lanes t and t^1 swap so that even t gets n = 4(t/2)..+3 (tile A) and
// odd t gets n = 8 + 4(t/2)..+3 (tile B).  Returns the 4-group index within the 16 (0..3).
__device__ __forceinline__ int pack16(const int (&dA)[3][4], const int (&dB)[3][4], int t, uint32_t (&word)[2]) {
    const bool odd = t & 1;
    // both tiles packed first (h = 0 pair in the low half, h = 1 pair in the high half), THEN one select per role
    const uint32_t pA = pack2(combine(dA[0][0], dA[1][0], dA[2][0]), combine(dA[0][1], dA[1][1], dA[2][1]),
                              pack2(combine(dA[0][2], dA[1][2], dA[2][2]), combine(dA[0][3], dA[1][3], dA[2][3]), 0));
    const uint32_t pB = pack2(combine(dB[0][0], dB[1][0], dB[2][0]), combine(dB[0][1], dB[1][1], dB[2][1]),
                              pack2(combine(dB[0][2], dB[1][2], dB[2][2]), combine(dB[0][3], dB[1][3], dB[2][3]), 0));
    const uint32_t keep = odd ? pB : pA;
    const uint32_t recv = __shfl_xor_sync(0xffffffffu, odd ? pA : pB, 1);
    // even lanes: own pair = n 4j, 4j+1 (low bytes), partner's = 4j+2, 4j+3 (high bytes); odd lanes the other way round
    const uint32_t lo = odd ? recv : keep, hi = odd ? keep : recv;
    word[0] = __byte_perm(lo, hi, 0x5410);
    word[1] = __byte_perm(lo, hi, 0x7632);
    return (t >> 1) + (odd ? 2 : 0);
}

// the same when only tile A carries data (the last 8 rows of a patch): even lanes still get 4 consecutive n of tile A,
// odd lanes' words are meaningless (n = 8..15 do not exist) and must not be used
__device__ __forceinline__ void pack8(const int (&dA)[3][4], int t, uint32_t (&word)[2]) {
    const uint32_t pA = pack2(combine(dA[0][0], dA[1][0], dA[2][0]), combine(dA[0][1], dA[1][1], dA[2][1]),
                              pack2(combine(dA[0][2], dA[1][2], dA[2][2]), combine(dA[0][3], dA[1][3], dA[2][3]), 0));
    const uint32_t recv = __shfl_xor_sync(0xffffffffu, pA, 1);
    word[0] = __byte_perm(pA, recv, 0x5410);
    word[1] = __byte_perm(pA, recv, 0x7632);
}

__device__ __forceinline__ void init_acc(int (&d)[3][4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) { d[0][i] = 1 << (kPrecisionBits - 1); d[1][i] = 0; d[2][i] = 0; }
}

// geometry of the block along the horizontal axis (shared by both passes: the V pass needs the column offset)
struct HGeo {
    int mt0, mt1, o_org, coff;
    __device__ __forceinline__ HGeo(const JobView& J) {
        const int oxb = J[USDU_J_OX_BASE];
        mt0 = max(oxb, 0) >> 4;
        mt1 = (min(oxb + BWX, J[USDU_J_N_OUT_H]) - 1) >> 4;
        o_org = min(oxb, mt0 << 4);            // output index of column 0 of the intermediate
        coff = 3 * (oxb - o_org);              // byte column of the intermediate that is block byte 0
    }
};

// ---- H pass: planes -> mid (row-packed) ---------------------------------------------------------------------------
template <int KS>
__device__ __forceinline__ void hpass(const uint8_t* __restrict__ planes, uint32_t* __restrict__ mid, const int32_t* __restrict__ tabs,
                                      const JobView& J, int PB, int plane_rows, int rows) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const FragTable F(tabs, J[USDU_J_ROWS_H]);
    const HGeo G(J);
    const int sx0 = J[USDU_J_IX0];
    const int full = rows >> 4;                                 // steps of 16 rows with both N-tiles
    const int tail = rows & 15;                                 // 1..8 rows left: tile A only; 9..15: one more full step
    const int steps = full + (tail > 8 ? 1 : 0);
    for (int mt = G.mt0 + w; mt <= G.mt1; mt += kT / 32) {
        uint32_t a[KS][3][4];
        F.load<KS>(a, mt, lane);
        const int krel = F.k0<KS>(mt) - sx0;                       // >= 0, multiple of 4
        uint32_t* mcol = mid + 3 * ((mt << 4) + g - G.o_org);
#pragma unroll 1
        for (int c = 0; c < 3; ++c) {
            const uint8_t* pa = planes + (size_t)c * plane_rows * PB + krel + 4 * t + g * PB;
            uint32_t* mo = mcol + c;
#pragma unroll 1
            for (int s = 0; s < steps; ++s, pa += 16 * PB, mo += 4 * MIDP) {
                int dA[3][4], dB[3][4];
                init_acc(dA); init_acc(dB);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) {
                    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(pa + 32 * ks), a1 = *reinterpret_cast<const uint32_t*>(pa + 32 * ks + 16);
                    const uint32_t b0 = *reinterpret_cast<const uint32_t*>(pa + 8 * PB + 32 * ks), b1 = *reinterpret_cast<const uint32_t*>(pa + 8 * PB + 32 * ks + 16);
                    mma_uu(dA[0], a[ks][0], a0, a1); mma_uu(dA[1], a[ks][1], a0, a1); mma_su(dA[2], a[ks][2], a0, a1);
                    mma_uu(dB[0], a[ks][0], b0, b1); mma_uu(dB[1], a[ks][1], b0, b1); mma_su(dB[2], a[ks][2], b0, b1);
                }
                uint32_t word[2];
                const int kg = pack16(dA, dB, t, word);          // 4 consecutive ROWS of outputs m = g (word 0) and g + 8 (word 1)
                mo[kg * MIDP] = word[0];
                mo[kg * MIDP + 24] = word[1];
            }
            if (tail >= 1 && tail <= 8) {                        // the last <= 8 rows: half the MMAs, half the recombination
                int dA[3][4];
                init_acc(dA);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) {
                    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(pa + 32 * ks), a1 = *reinterpret_cast<const uint32_t*>(pa + 32 * ks + 16);
                    mma_uu(dA[0], a[ks][0], a0, a1); mma_uu(dA[1], a[ks][1], a0, a1); mma_su(dA[2], a[ks][2], a0, a1);
                }
                uint32_t word[2];
                pack8(dA, t, word);
                if (!(t & 1)) {                                  // rows 4 (t/2) .. + 3 of this last group of 8
                    mo[(t >> 1) * MIDP] = word[0];
                    mo[(t >> 1) * MIDP + 24] = word[1];
                }
            }
        }
    }
}

// ---- V pass: mid -> 4-byte strips of block rows, handed to an epilogue -----------------------------------------------
// Epilogue::rows(r0, r1) fixes the two block rows of the M-tile's halves (m = g and g + 8) once per M-tile;
// Epilogue::prefetch(strip) issues the loads the epilogue will need BEFORE the MMAs;
// Epilogue::store(pre, h, strip, word) consumes them (bytes 4 strip .. 4 strip + 3 of row half h).
template <int KS, class Epilogue>
__device__ __forceinline__ void vpass(const uint32_t* __restrict__ mid, const int32_t* __restrict__ tabs, const JobView& J, int bh,
                                      Epilogue& epi) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const FragTable F(tabs, J[USDU_J_ROWS_V]);
    const HGeo G(J);
    const int oyb = J[USDU_J_OY_BASE], sy0 = J[USDU_J_IY0];
    const int mv0 = max(oyb, 0) >> 4, mv1 = (min(oyb + bh, J[USDU_J_N_OUT_V]) - 1) >> 4;
    constexpr int PAIRS = BWX * 3 / 16;                        // 24 pairs of N-tiles = 384 byte columns: 3 per warp
    const int sub = (t >> 1) + ((t & 1) ? 2 : 0);               // which 4-byte strip of the pair this lane ends with
#pragma unroll 1
    for (int mv = mv0; mv <= mv1; ++mv) {
        uint32_t a[KS][3][4];
        F.load<KS>(a, mv, lane);
        const int r0 = (mv << 4) + g - oyb;                     // block row of output m = g; m = g + 8 is r0 + 8
        epi.rows(r0, r0 + 8);
        const uint32_t* mp = mid + (((F.k0<KS>(mv) - sy0) >> 2) + t) * MIDP + G.coff + g + 16 * w;
        int strip = 4 * w + sub;
#pragma unroll 1
        for (int p = w; p < PAIRS; p += kT / 32, mp += 16 * (kT / 32), strip += 4 * (kT / 32)) {
            const typename Epilogue::Pre pre = epi.prefetch(strip);
            int dA[3][4], dB[3][4];
            init_acc(dA); init_acc(dB);
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                const uint32_t a0 = mp[(8 * ks) * MIDP], a1 = mp[(8 * ks + 4) * MIDP];
                const uint32_t b0 = mp[(8 * ks) * MIDP + 8], b1 = mp[(8 * ks + 4) * MIDP + 8];
                mma_uu(dA[0], a[ks][0], a0, a1); mma_uu(dA[1], a[ks][1], a0, a1); mma_su(dA[2], a[ks][2], a0, a1);
                mma_uu(dB[0], a[ks][0], b0, b1); mma_uu(dB[1], a[ks][1], b0, b1); mma_su(dB[2], a[ks][2], b0, b1);
            }
            uint32_t word[2];
            pack16(dA, dB, t, word);                            // 4 consecutive BYTES of block rows r0 (word 0) and r0 + 8 (word 1)
            epi.store(pre, 0, strip, word[0]);
            epi.store(pre, 1, strip, word[1]);
        }
    }
}

// ---- staging: interleaved source -> three byte planes ------------------------------------------------------------------
// planes[c][row][x]: row pitch PB, plane_rows rows per plane.  A unit = (row, chunk of 4 pixels).
__device__ __forceinline__ void store_planes(uint8_t* planes, int PB, int plane_rows, int r, int ch, uint32_t R, uint32_t G, uint32_t B) {
    uint8_t* p = planes + (size_t)r * PB + 4 * ch;
    *reinterpret_cast<uint32_t*>(p) = R;
    *reinterpret_cast<uint32_t*>(p + (size_t)plane_rows * PB) = G;
    *reinterpret_cast<uint32_t*>(p + (size_t)2 * plane_rows * PB) = B;
}

// 12 interleaved bytes (w0 w1 w2) -> R G B words of 4 pixels
__device__ __forceinline__ void deinterleave(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t& R, uint32_t& G, uint32_t& B) {
    R = __byte_perm(__byte_perm(w0, w1, 0x0630), w2, 0x5210);      // bytes 0 3 6 9
    G = __byte_perm(__byte_perm(w0, w1, 0x0741), w2, 0x6210);      // bytes 1 4 7 10
    B = __byte_perm(__byte_perm(w0, w1, 0x0052), w2, 0x7410);      // bytes 2 5 8 11
}

// i / d for 0 <= i < 2^16, 1 <= d < 2^16 without a division: m = floor(2^32 / d) + 1
// (d == 1 wraps m to 0, which stands for "i itself")
__device__ __forceinline__ uint32_t recip_u16(int d) { return 0xFFFFFFFFu / (uint32_t)d + 1u; }
__device__ __forceinline__ int div_u16(int i, uint32_t m) { return m ? (int)__umulhi((uint32_t)i, m) : i; }

// fp32 source in [0,1] (sampler output): Q1 truncation on the fly.  src -> first float of the staged patch.
// kU units per thread per trip, every load issued before the first use (12 x 16 bytes in flight per thread).
// Evict-first loads (__ldcs): the sampler output is dead once blended, so its lines should leave L2 before the next wave's
// crop output, which the next sampler reads (DESIGN section 9.1).
__device__ __forceinline__ void stage_f32(uint8_t* planes, int PB, int plane_rows, const float* __restrict__ src, int64_t pitch_f,
                                          int rows, int cols) {
    constexpr int kU = 4;                       // 1024 units per trip: a 128 x 16 block (<= 825 units) is staged in ONE round of loads
    const int chunks = cols >> 2, total = rows * chunks;
    const uint32_t rc = recip_u16(chunks);
    for (int i0 = threadIdx.x; i0 < total; i0 += kT * kU) {
        float4 f[kU][3];
        int rr[kU], cc[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int i = min(i0 + u * kT, total - 1);
            rr[u] = div_u16(i, rc); cc[u] = i - rr[u] * chunks;
            const float4* p = reinterpret_cast<const float4*>(src + (int64_t)rr[u] * pitch_f) + cc[u] * 3;
            f[u][0] = __ldcs(p); f[u][1] = __ldcs(p + 1); f[u][2] = __ldcs(p + 2);
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            if (i0 + u * kT >= total) break;
            const float4 f0 = f[u][0], f1 = f[u][1], f2 = f[u][2];
            const uint32_t R = quant_u8(f0.x) | (quant_u8(f0.w) << 8) | (quant_u8(f1.z) << 16) | (quant_u8(f2.y) << 24);
            const uint32_t G = quant_u8(f0.y) | (quant_u8(f1.x) << 8) | (quant_u8(f1.w) << 16) | (quant_u8(f2.z) << 24);
            const uint32_t B = quant_u8(f0.z) | (quant_u8(f1.y) << 8) | (quant_u8(f2.x) << 16) | (quant_u8(f2.w) << 24);
            store_planes(planes, PB, plane_rows, rr[u], cc[u], R, G, B);
        }
    }
}

// u8 interleaved source in global memory (transport payload, canvas without TMA); src 4-byte aligned
__device__ __forceinline__ void stage_u8(uint8_t* planes, int PB, int plane_rows, const uint8_t* __restrict__ src, int64_t pitch,
                                         int rows, int cols) {
    constexpr int kU = 4;
    const int chunks = cols >> 2, total = rows * chunks;
    const uint32_t rc = recip_u16(chunks);
    for (int i0 = threadIdx.x; i0 < total; i0 += kT * kU) {
        uint32_t w[kU][3];
        int rr[kU], cc[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int i = min(i0 + u * kT, total - 1);
            rr[u] = div_u16(i, rc); cc[u] = i - rr[u] * chunks;
            const uint32_t* p = reinterpret_cast<const uint32_t*>(src + (int64_t)rr[u] * pitch) + cc[u] * 3;
            w[u][0] = __ldg(p); w[u][1] = __ldg(p + 1); w[u][2] = __ldg(p + 2);
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            if (i0 + u * kT >= total) break;
            uint32_t R, G, B;
            deinterleave(w[u][0], w[u][1], w[u][2], R, G, B);
            store_planes(planes, PB, plane_rows, rr[u], cc[u], R, G, B);
        }
    }
}

// the same from the two TMA boxes in shared memory (virtual 512-byte rows); lead_b = bytes before the first pixel
__device__ __forceinline__ void stage_raw(uint8_t* planes, int PB, int plane_rows, const uint8_t* raw, int rows, int cols, int lead_b) {
    const int chunks = cols >> 2;
    const uint32_t rc = recip_u16(chunks);
    for (int i = threadIdx.x; i < rows * chunks; i += kT) {
        const int r = div_u16(i, rc), ch = i - r * chunks;
        uint32_t w[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int o = lead_b + 12 * ch + 4 * k;
            w[k] = *reinterpret_cast<const uint32_t*>(raw + (size_t)(o >> 8) * (kBoxR * kBoxB) + r * kBoxB + (o & 255));
        }
        uint32_t R, G, B;
        deinterleave(w[0], w[1], w[2], R, G, B);
        store_planes(planes, PB, plane_rows, r, ch, R, G, B);
    }
}

// KSMAX = 1: every axis of the launch fits one k-step (scales up to ~1.4): no two-step code, fewer registers
template <int KSMAX, class Epilogue>
__device__ __forceinline__ void both_passes(const uint8_t* planes, uint32_t* mid, const int32_t* tabs, const JobView& J, int PB,
                                            int plane_rows, int bh, Epilogue& epi) {
    const int rows = J[USDU_J_ROWS];
    if (KSMAX == 1 || J[USDU_J_TAPS_H] <= 1) hpass<1>(planes, mid, tabs, J, PB, plane_rows, rows);
    else hpass<KSMAX>(planes, mid, tabs, J, PB, plane_rows, rows);
    __syncthreads();
    if (KSMAX == 1 || J[USDU_J_TAPS_V] <= 1) vpass<1>(mid, tabs, J, bh, epi);
    else vpass<KSMAX>(mid, tabs, J, bh, epi);
}

// ======================================================================================
// crop + resize
// ======================================================================================
struct CropEpilogue {
    float* dst;          // &out[tile][b][oy0][ox0][0]
    int64_t row_pitch;   // floats per output row
    int ow3, rows_out;
    float* rp[2];        // row pointers of the current M-tile halves (nullptr = row outside the block)
    struct Pre {};
    __device__ __forceinline__ void rows(int r0, int r1) {
        rp[0] = (r0 >= 0 && r0 < rows_out) ? dst + (int64_t)r0 * row_pitch : nullptr;
        rp[1] = (r1 >= 0 && r1 < rows_out) ? dst + (int64_t)r1 * row_pitch : nullptr;
    }
    __device__ __forceinline__ Pre prefetch(int) const { return Pre{}; }
    __device__ __forceinline__ void store(const Pre&, int h, int strip, uint32_t v) {
        if (rp[h] != nullptr && 4 * strip < ow3) {   // ow3 is a multiple of 4 (pw % 8 == 0)
            // u / 255.0f in arithmetic (dequant_u8_fast): a 256-entry table in shared memory costs 4 data-dependent loads per
            // thread that collide on banks -- 78 % of the kernel's excess shared-memory wavefronts in the r02e profile
            float4 o;
            o.x = dequant_u8_fast(v & 0xFF); o.y = dequant_u8_fast((v >> 8) & 0xFF);
            o.z = dequant_u8_fast((v >> 16) & 0xFF); o.w = dequant_u8_fast(v >> 24);
            store_handoff(rp[h] + 4 * strip, o);
        }
    }
};

// kSrc: 0 = u8 canvas read with LDG, 1 = u8 canvas staged by TMA, 2 = the fp32 IMAGE itself (`canvas` is then a float
// pointer and `pitch` counts floats per row): Q0's truncating cast happens while staging, the window is bit-identical
// to cropping the quantised canvas -- a rank of a conflict-free partition never needs the quantised canvas at all.
template <int kSrc, int KSMAX, int kOcc>
__global__ void __launch_bounds__(kT, KSMAX == 1 ? kOcc : 3)
crop_mma_kernel(const uint8_t* __restrict__ canvas, int H, int64_t pitch, const int32_t* __restrict__ tabs,
                const int32_t* __restrict__ jobs, float* __restrict__ out, int patch_w, int plane_rows, int mid_rows, int W3,
                const __grid_constant__ CUtensorMap cmap) {
    extern __shared__ __align__(128) uint8_t smem[];
    // [mid | raw (TMA boxes), aliased: raw is dead before the H pass writes mid] [job] [bar] [planes]
    constexpr bool kTma = kSrc == 1;
    const size_t region = kTma ? max(mid_bytes(mid_rows), (size_t)2 * kBoxR * kBoxB) : mid_bytes(mid_rows);   // (boxes are always 48 rows)
    uint32_t* mid = reinterpret_cast<uint32_t*>(smem);
    uint8_t* raw = smem;
    int32_t* job_sm = reinterpret_cast<int32_t*>(smem + region);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + region + kHeadBytes);
    uint8_t* planes = smem + region + kHeadBytes + 16;
    const int PB = plane_pitch(patch_w);
    pdl_launch_dependents();
    load_job(job_sm, jobs, blockIdx.x);
    if (kTma && threadIdx.x == 0) tma::mbar_init(bar, 1);
    __syncthreads();
    const JobView J{job_sm};
    const int b = blockIdx.y;
    pdl_wait();                                // the canvas is the previous kernel's output
    const int sa3 = J[USDU_J_SRC_A] * 3;
    if (kTma) {
        if (threadIdx.x == 0) {
            const int x = sa3 & ~15, y = J[USDU_J_SRC_B];                          // 16-byte aligned box start
            const bool two = (sa3 - x) + J[USDU_J_COLS] * 3 > kBoxB && x + kBoxB < W3;
            tma::mbar_expect_tx(bar, (two ? 2 : 1) * kBoxR * kBoxB);
            tma::load_3d(raw, &cmap, x, y, b, bar);
            if (two) tma::load_3d(raw + kBoxR * kBoxB, &cmap, x + kBoxB, y, b, bar);
        }
        tma::mbar_wait(bar, 0);
        stage_raw(planes, PB, plane_rows, raw, J[USDU_J_ROWS], J[USDU_J_COLS], sa3 & 15);
    } else if (kSrc == 2) {
        const float* src = reinterpret_cast<const float*>(canvas) + ((int64_t)b * H + J[USDU_J_SRC_B]) * pitch + sa3;
        stage_f32(planes, PB, plane_rows, src, pitch, J[USDU_J_ROWS], J[USDU_J_COLS]);
    } else {
        const uint8_t* src = canvas + ((int64_t)b * H + J[USDU_J_SRC_B]) * pitch + sa3;
        stage_u8(planes, PB, plane_rows, src, pitch, J[USDU_J_ROWS], J[USDU_J_COLS]);
    }
    __syncthreads();                           // planes complete; raw (aliased with mid) is dead
    CropEpilogue epi;
    epi.row_pitch = J[USDU_J_PITCH];
    epi.dst = out + J.i64(USDU_J_OFF_LO) + (int64_t)b * J.i64(USDU_J_FRAME_LO) + (int64_t)J[USDU_J_DST_Y] * epi.row_pitch +
              (int64_t)J[USDU_J_DST_X] * 3;
    epi.ow3 = J[USDU_J_COLS_OUT] * 3;
    epi.rows_out = J[USDU_J_ROWS_OUT];
    both_passes<KSMAX>(planes, mid, tabs, J, PB, plane_rows, J[USDU_J_CY1], epi);
}

// ======================================================================================
// blend
// ======================================================================================
struct DTile {
    uint8_t* base;
    int bh;                                  // rows per box
    // byte offset of strip `strip` inside a row of the two-box block (box 1 starts bh * 192 bytes after box 0)
    __device__ __forceinline__ int strip_off(int strip) const {
        return 4 * strip + (strip >= kDBox / 4 ? bh * kDBox - kDBox : 0);
    }
};

// interior of a tile (alpha == 255 over the whole block): the canvas block becomes S
struct BlendOpaque {
    DTile d;
    int nrows;
    uint8_t* rp[2];
    struct Pre {};
    __device__ __forceinline__ void rows(int r0, int r1) {
        rp[0] = (r0 >= 0 && r0 < nrows) ? d.base + r0 * kDBox : nullptr;
        rp[1] = (r1 >= 0 && r1 < nrows) ? d.base + r1 * kDBox : nullptr;
    }
    __device__ __forceinline__ Pre prefetch(int) const { return Pre{}; }
    __device__ __forceinline__ void store(const Pre&, int h, int strip, uint32_t v) {
        if (rp[h] != nullptr) *reinterpret_cast<uint32_t*>(rp[h] + d.strip_off(strip)) = v;
    }
};

// general case: per-pixel alpha from the feather template, zero outside the tile's sub-rect
struct BlendFeather {
    DTile d;
    const uint8_t* mask;   // template address of block pixel (0,0) (may point outside; guarded by the rect)
    int mpitch;
    int cx0, cx1, cy0, cy1;   // sub-rect in block pixel coordinates
    uint8_t* rp[2];           // canvas-block rows of the current M-tile halves (nullptr = outside [cy0, cy1))
    const uint8_t* mp[2];     // their template rows
    struct Pre {
        uint32_t aa[2], ab[2];   // per row half: alpha of the two pixels the 4 bytes touch
        int split;               // bytes [0, split) belong to the first pixel
    };
    __device__ __forceinline__ void rows(int r0, int r1) {
        const bool in0 = r0 >= cy0 && r0 < cy1, in1 = r1 >= cy0 && r1 < cy1;
        rp[0] = in0 ? d.base + r0 * kDBox : nullptr;
        rp[1] = in1 ? d.base + r1 * kDBox : nullptr;
        mp[0] = mask + (int64_t)r0 * mpitch;
        mp[1] = mask + (int64_t)r1 * mpitch;
    }
    __device__ __forceinline__ Pre prefetch(int strip) const {
        const int col = 4 * strip;
        const int pa = col / 3, pb = (col + 3) / 3;          // pb = pa or pa + 1
        const bool ina = pa >= cx0 && pa < cx1, inb = pb >= cx0 && pb < cx1;
        Pre p;
        p.split = 3 * pb - col;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            p.aa[h] = (rp[h] != nullptr && ina) ? (uint32_t)__ldg(mp[h] + pa) : 0u;
            p.ab[h] = (rp[h] != nullptr && inb) ? (uint32_t)__ldg(mp[h] + pb) : 0u;
        }
        return p;
    }
    __device__ __forceinline__ void store(const Pre& p, int h, int strip, uint32_t v) {
        const uint32_t aa = p.aa[h], ab = p.ab[h];
        if ((aa | ab) == 0u) return;                         // also: rows outside [cy0, cy1)
        uint32_t* w = reinterpret_cast<uint32_t*>(rp[h] + d.strip_off(strip));
        if ((aa & ab) == 255u) { *w = v; return; }
        const uint32_t dv = *w;
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t a = i < p.split ? aa : ab;
            o |= composite8((v >> (8 * i)) & 0xFF, (dv >> (8 * i)) & 0xFF, a) << (8 * i);
        }
        *w = o;
    }
};

template <bool kSrcU8, int KSMAX>
__global__ void __launch_bounds__(kT, kOccSmall)
blend_mma_kernel(const int32_t* __restrict__ tabs, const uint8_t* __restrict__ mask_pool, const int32_t* __restrict__ jobs,
                 const void* __restrict__ src_v, int W3, int patch_w, int plane_rows, int mid_rows, int block_rows,
                 const __grid_constant__ CUtensorMap cmap) {
    extern __shared__ __align__(128) uint8_t smem[];
    // [canvas block: 2 boxes x block_rows x 192] [job] [bar] [mid] [planes]   (planes BEHIND mid: the vertical K windows may
    // read a few row groups past the rows the horizontal pass wrote -- zero coefficients -- and must stay inside the CTA's memory)
    const size_t dbytes = (size_t)2 * block_rows * kDBox;
    int32_t* job_sm = reinterpret_cast<int32_t*>(smem + dbytes);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + dbytes + kHeadBytes);
    uint32_t* mid = reinterpret_cast<uint32_t*>(smem + dbytes + kHeadBytes + 16);
    uint8_t* planes = smem + dbytes + kHeadBytes + 16 + mid_bytes(mid_rows);
    const int PB = plane_pitch(patch_w);
    const int b = blockIdx.y;
    const JobView J{job_sm};
    DTile D{smem, block_rows};
    int idx = blockIdx.x;
    pdl_launch_dependents();
    load_job(job_sm, jobs, idx);
    if (threadIdx.x == 0) tma::mbar_init(bar, 1);
    __syncthreads();
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
            __syncthreads();                   // the previous tile's passes are done with job / planes / mid
            load_job(job_sm, jobs, idx);
            __syncthreads();
        }
        const int64_t first_el = J.i64(USDU_J_SRC_A) + (int64_t)b * J.i64(USDU_J_FRAME_LO);
        if (kSrcU8)
            stage_u8(planes, PB, plane_rows, static_cast<const uint8_t*>(src_v) + first_el, J[USDU_J_PITCH], J[USDU_J_ROWS], J[USDU_J_COLS]);
        else
            stage_f32(planes, PB, plane_rows, static_cast<const float*>(src_v) + first_el, J[USDU_J_PITCH], J[USDU_J_ROWS], J[USDU_J_COLS]);
        __syncthreads();
        if (first) tma::mbar_wait(bar, 0);     // the canvas block has landed (before any epilogue touches it)
        if (J[USDU_J_FLAGS] & 1) {
            BlendOpaque epi;
            epi.d = D;
            epi.nrows = J[USDU_J_ROWS_OUT];
            both_passes<KSMAX>(planes, mid, tabs, J, PB, plane_rows, block_rows, epi);
        } else {
            BlendFeather epi;
            epi.d = D;
            epi.mpitch = J[USDU_J_MPITCH];
            epi.mask = mask_pool + J.i64(USDU_J_OFF_LO);
            epi.cx0 = J[USDU_J_CX0]; epi.cx1 = J[USDU_J_CX1];
            epi.cy0 = J[USDU_J_CY0]; epi.cy1 = J[USDU_J_CY1];
            both_passes<KSMAX>(planes, mid, tabs, J, PB, plane_rows, block_rows, epi);
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
        tma::store_wait_read();
    }
}

static size_t crop_smem(int patch_w, int plane_rows, int mid_rows, bool use_tma) {
    const size_t region = use_tma ? max(mid_bytes(mid_rows), (size_t)2 * kBoxR * kBoxB) : mid_bytes(mid_rows);
    return region + kHeadBytes + 16 + planes_bytes(patch_w, plane_rows);
}
static size_t blend_smem(int patch_w, int plane_rows, int mid_rows, int block_rows) {
    return (size_t)2 * block_rows * kDBox + kHeadBytes + 16 + planes_bytes(patch_w, plane_rows) + mid_bytes(mid_rows);
}

static int optin(const void* fn, size_t bytes) {
    if (bytes > 227 * 1024) {
        set_error("tensor-core kernel needs %zu bytes of shared memory (> 227 KB)", bytes);
        return USDU_ERR_UNSUPPORTED;
    }
    return raise_smem_limit(fn, bytes);
}

static int split_patch_h(int patch_h, int* plane_rows, int* mid_rows, const char* who) {
    *plane_rows = patch_h & 0xFFFF;
    *mid_rows = (patch_h >> 16) & 0xFFFF;
    if (*plane_rows <= 0 || *plane_rows % 8 || *mid_rows < *plane_rows || *mid_rows % 4) {
        set_error("%s: with USDU_FLAG_MMA patch_h carries plane rows (x8) in bits 0..15 and intermediate rows (x4, >= plane rows) "
                  "in bits 16..31; got %d / %d", who, *plane_rows, *mid_rows);
        return USDU_ERR_INVALID;
    }
    return USDU_OK;
}

template <class K, class... Args>
static int launch_one(K kernel, size_t smem, dim3 grid, cudaStream_t st, Args... args) {
    int s = optin((const void*)kernel, smem);
    if (s != USDU_OK) return s;
    USDU_CUDA(launch_pdl(kernel, grid, dim3(kT), smem, st, args...));
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int launch_crop(const void* canvas, int src_f32, int B, int H, int W, int64_t pitch, const int32_t* tabs, const int32_t* items,
                int n_items, int patch_w, int patch_h, float* out, int two_ksteps, cudaStream_t st) {
    int plane_rows, mid_rows;
    int s = split_patch_h(patch_h, &plane_rows, &mid_rows, "usdu_tile_crop_resize");
    if (s != USDU_OK) return s;
    CUtensorMap cmap;
    memset(&cmap, 0, sizeof(cmap));
    const uint8_t* cv = static_cast<const uint8_t*>(canvas);
    const dim3 grid(n_items, B);
    const int W3 = W * 3;
    const bool large = (int64_t)n_items * B >= (int64_t)kLargeGridPerSM * grid_sms() && !two_ksteps;
#define USDU_CROP_LAUNCH(SRC)                                                                                                                   \
    (two_ksteps ? launch_one(crop_mma_kernel<SRC, 2, kOccSmall>, smem, grid, st, cv, H, pitch, tabs, items, out, patch_w, plane_rows, mid_rows, W3, cmap) \
     : large    ? launch_one(crop_mma_kernel<SRC, 1, kOccLarge>, smem, grid, st, cv, H, pitch, tabs, items, out, patch_w, plane_rows, mid_rows, W3, cmap) \
                : launch_one(crop_mma_kernel<SRC, 1, kOccSmall>, smem, grid, st, cv, H, pitch, tabs, items, out, patch_w, plane_rows, mid_rows, W3, cmap))
    if (src_f32) {
        if (W % 4 != 0 || ((uintptr_t)canvas & 15) != 0) {
            set_error("usdu_tile_crop_resize_f32: the image width must be a multiple of 4 and the image 16-byte aligned");
            return USDU_ERR_UNSUPPORTED;
        }
        const size_t smem = crop_smem(patch_w, plane_rows, mid_rows, false);
        return USDU_CROP_LAUNCH(2);
    }
    // TMA staging needs the patch to fit the two boxes (the planner keeps the staged rows <= 48 for scales <= ~1.2)
    bool use_tma = plane_rows <= kBoxR && 12 + patch_w * 3 <= 2 * kBoxB && ((uintptr_t)canvas & 15) == 0;
    if (use_tma) use_tma = tma::encode_u8_3d(&cmap, canvas, (uint64_t)W * 3, (uint64_t)H, (uint64_t)B, (uint64_t)pitch, kBoxB, kBoxR);
    const size_t smem = crop_smem(patch_w, plane_rows, mid_rows, use_tma);
    if (use_tma) return USDU_CROP_LAUNCH(1);
    return USDU_CROP_LAUNCH(0);
#undef USDU_CROP_LAUNCH
}

int launch_blend(uint8_t* canvas, int B, int H, int W, int64_t pitch, const int32_t* tabs, const uint8_t* mask_pool,
                 const int32_t* items, int n_items, int patch_w, int patch_h, const void* src, int src_is_u8, int block_rows,
                 int two_ksteps, cudaStream_t st) {
    if (block_rows != 16 && block_rows != 32) {
        set_error("usdu_tile_blend: the tensor-core path needs a block height of 16 or 32 in flags bits 8..15, got %d", block_rows);
        return USDU_ERR_INVALID;
    }
    int plane_rows, mid_rows;
    int s = split_patch_h(patch_h, &plane_rows, &mid_rows, "usdu_tile_blend");
    if (s != USDU_OK) return s;
    CUtensorMap cmap;
    memset(&cmap, 0, sizeof(cmap));
    if (((uintptr_t)canvas & 15) != 0 ||
        !tma::encode_u8_3d(&cmap, canvas, (uint64_t)W * 3, (uint64_t)H, (uint64_t)B, (uint64_t)pitch, kDBox, block_rows)) {
        set_error("usdu_tile_blend: cannot build the canvas tensor map (cuTensorMapEncodeTiled)");
        return USDU_ERR_CUDA;
    }
    const size_t smem = blend_smem(patch_w, plane_rows, mid_rows, block_rows);
    const dim3 grid(n_items, B);
    const int W3 = W * 3;
    if (src_is_u8)
        return two_ksteps ? launch_one(blend_mma_kernel<true, 2>, smem, grid, st, tabs, mask_pool, items, src, W3, patch_w, plane_rows, mid_rows, block_rows, cmap)
                          : launch_one(blend_mma_kernel<true, 1>, smem, grid, st, tabs, mask_pool, items, src, W3, patch_w, plane_rows, mid_rows, block_rows, cmap);
    return two_ksteps ? launch_one(blend_mma_kernel<false, 2>, smem, grid, st, tabs, mask_pool, items, src, W3, patch_w, plane_rows, mid_rows, block_rows, cmap)
                      : launch_one(blend_mma_kernel<false, 1>, smem, grid, st, tabs, mask_pool, items, src, W3, patch_w, plane_rows, mid_rows, block_rows, cmap);
}

// Resident CTAs per SM of the build launch_crop / launch_blend would pick (kernel = USDU_KERNEL_*, the crop's
// USDU_KERNEL_LARGE bit as kLargeGridPerSM decides it) at the dynamic shared memory it would request for these patch
// words.  use_device: cudaOccupancyMaxActiveBlocksPerMultiprocessor on the current device; else the table of the
// launch bounds (kOccSmall / kOccLarge, which ptxas meets: 80 / 64 registers at most) and 228 KB of shared memory per
// SM, 1 KB of it reserved per CTA.  0 when the build does not fit an SM, a negative usdu_status on an error.
int resident_ctas(int kernel, bool two_ksteps, int patch_w, int patch_h, int block_rows, bool use_device) {
    const int plane_rows = patch_h & 0xFFFF, mid_rows = (patch_h >> 16) & 0xFFFF;
    const int base = kernel & ~USDU_KERNEL_LARGE;
    const bool large = (kernel & USDU_KERNEL_LARGE) && base != USDU_KERNEL_BLEND && !two_ksteps;
    size_t smem;
    const void* fn;
    if (base == USDU_KERNEL_BLEND) {
        smem = blend_smem(patch_w, plane_rows, mid_rows, block_rows);
        fn = two_ksteps ? (const void*)blend_mma_kernel<false, 2> : (const void*)blend_mma_kernel<false, 1>;
    } else if (base == USDU_KERNEL_CROP_LDG || base == USDU_KERNEL_CROP_TMA) {
        const bool tma = base == USDU_KERNEL_CROP_TMA;
        smem = crop_smem(patch_w, plane_rows, mid_rows, tma);
        fn = two_ksteps ? (tma ? (const void*)crop_mma_kernel<1, 2, kOccSmall> : (const void*)crop_mma_kernel<0, 2, kOccSmall>)
             : large    ? (tma ? (const void*)crop_mma_kernel<1, 1, kOccLarge> : (const void*)crop_mma_kernel<0, 1, kOccLarge>)
                        : (tma ? (const void*)crop_mma_kernel<1, 1, kOccSmall> : (const void*)crop_mma_kernel<0, 1, kOccSmall>);
    } else {
        set_error("usdu_mma_resident_ctas: unknown kernel %d", kernel);
        return USDU_ERR_INVALID;
    }
    if (smem > 227 * 1024) return 0;
    if (!use_device) {
        const size_t per_cta = (smem + 1024 + 127) / 128 * 128;
        return (int)std::min((size_t)(large ? kOccLarge : kOccSmall), (size_t)228 * 1024 / per_cta);
    }
    int s = raise_smem_limit(fn, smem);
    if (s != USDU_OK) return s;
    int n = 0;
    USDU_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, kT, smem));
    return n;
}

}  // namespace mma
}  // namespace usdu

int usdu_mma_resident_ctas(int kernel, int two_ksteps, int patch_w, int patch_h, int block_rows, int use_device) {
    if (patch_w <= 0 || (patch_h & 0xFFFF) <= 0 || ((patch_h >> 16) & 0xFFFF) < (patch_h & 0xFFFF) || block_rows < 0 ||
        block_rows > USDU_FAST_BLOCK_H) {
        usdu::set_error("usdu_mma_resident_ctas: bad patch (w=%d h=%#x) or block height %d", patch_w, patch_h, block_rows);
        return USDU_ERR_INVALID;
    }
    return usdu::mma::resident_ctas(kernel, two_ksteps != 0, patch_w, patch_h, block_rows, use_device != 0);
}
