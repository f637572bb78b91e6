// usdu_fast.cuh -- the two-pass 8-bit LANCZOS engine shared by the fast crop and blend
// kernels (sm_90a).
//
// Cost model (tools/ubench/pipes.cu measures it): IMAD issues at 64 lanes/clk/SM, byte
// extraction (PRMT) at 64, and every instruction takes one of the 128 issue slots/clk/SM.
// The naive form -- one shared-memory byte load + one IMAD per tap -- needs ~300 thread
// instructions per output byte.  Here one 32-bit shared-memory load brings the tap's byte
// of FOUR independent lines (rows in the H pass, byte columns in the V pass), so a tap costs
// 1/4 LDS + PRMT + IMAD per byte, registers stay <= 64 and no dynamic register indexing is
// needed.  (A register-window variant with a warp-uniform switch needs more instructions per
// byte and dynamic register indexing; this form is simpler.)
//
//   H pass  thread = output pixel column (coefficients in registers), loop over (group of 4
//           rows, channel).  Input is staged PLANAR and ROW-PACKED: word(g, c, x) = bytes of
//           rows 4g..4g+3 of channel c at pixel x, so tap t of 4 rows is ONE LDS.32 and one
//           PRMT per row; no alignment fix-ups, consecutive lanes read consecutive words.
//   V pass  item = (output row, 4-byte column strip); tap t of 4 byte columns is one LDS.32 of
//           `mid` (row-major u8, pixel interleaved, block pixel coordinates).
//
// Arithmetic is Pillow's (Resample.c): acc = 2^21 + sum in*k ; out = clip8(acc >> 22), with a
// u8 intermediate between the passes.
#pragma once
#include "usdu_common.cuh"

namespace usdu {
namespace fast {

constexpr int kT = 256;                    // threads per CTA: 2 sub-groups of FBW threads
constexpr int FBW = USDU_FAST_BLOCK_W;     // 128-pixel wide blocks
constexpr int FBH = USDU_FAST_BLOCK_H;     // up to 32 rows
constexpr int MAXTAPS = USDU_FAST_TAPS_WIDE;   // 15: the wide variant, picked per job and axis
constexpr int R = 4;                       // independent lines (rows / byte columns) per thread
constexpr int MID_PITCH = FBW * 3 + 4;     // 388 bytes: 4 consecutive rows land 4 banks apart

// one output of an axis: first input index + TAPS coefficients (TAPS + 1 int32, 16-byte aligned)
template <int TAPS>
struct PackedRow {
    int first;
    int k[TAPS];
};

template <int TAPS, class LoadInt4>
__device__ __forceinline__ PackedRow<TAPS> read_row(LoadInt4 ld) {
    PackedRow<TAPS> r;
    int v[TAPS + 1];
#pragma unroll
    for (int i = 0; i < (TAPS + 1) / 4; ++i) {
        const int4 q = ld(i);
        v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
    }
    r.first = v[0];
#pragma unroll
    for (int t = 0; t < TAPS; ++t) r.k[t] = v[t + 1];
    return r;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// clip8(acc >> 22) in two instructions (SHF + VIMNMX.RELU)
__device__ __forceinline__ uint32_t finish(int acc) {
    return (uint32_t)__vimin_s32_relu(acc >> kPrecisionBits, 255);
}

// 4 lines x N taps: words w[t] hold the 4 lines' bytes of tap t.  N <= TAPS is the number of taps
// the axis really uses (an up-scaling LANCZOS axis has exactly 6: int(c+3.5) - int(c-2.5); the
// 7th slot of its packed row is always 0 and is not multiplied).
template <int TAPS, int N>
__device__ __forceinline__ void dot4(const uint32_t (&w)[N], const PackedRow<TAPS>& row, int (&acc)[R]) {
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 1 << (kPrecisionBits - 1);
#pragma unroll
    for (int t = 0; t < N; ++t) {
        // (moving one of the four extractions to the integer-FMA pipe with IMAD.HI -- hi32(w*2^8)
        // == w >> 24 -- would put more work on the already busier IMAD pipe)
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] += (int)__byte_perm(w[t], 0, 0x4440 + r) * row.k[t];
    }
}

// The job record, staged in shared memory (warp-uniform reads).
struct JobView {
    const int32_t* j;
    __device__ __forceinline__ int operator[](int i) const { return j[i]; }
    __device__ __forceinline__ int64_t i64(int lo) const {
        return (int64_t)(uint32_t)j[lo] | ((int64_t)j[lo + 1] << 32);
    }
};

// ---- H pass: in (planar, row packed) -> mid[row][block px * 3 + c] ----------------------
// `row` = this thread's pixel column coefficients (loaded from global before staging).
template <int TAPS, int N = TAPS>
__device__ __forceinline__ void hpass(const uint32_t* __restrict__ in, uint8_t* __restrict__ mid, const PackedRow<TAPS>& row,
                                      int ix0, int rows_in, int xw) {
    const int px = threadIdx.x % FBW, sub = threadIdx.x / FBW;
    const uint32_t* w0 = in + (row.first - ix0);
    const int units = ((rows_in + 3) >> 2) * 3;
    uint8_t* o = mid + px * 3;
#pragma unroll 2
    for (int u = sub; u < units; u += kT / FBW) {
        const uint32_t* wp = w0 + (size_t)u * xw;
        uint32_t w[N];
#pragma unroll
        for (int t = 0; t < N; ++t) w[t] = wp[t];
        int acc[R];
        dot4<TAPS, N>(w, row, acc);
        const int g = u / 3, c = u - g * 3;
        uint8_t* oo = o + (size_t)(4 * g) * MID_PITCH + c;
#pragma unroll
        for (int r = 0; r < R; ++r) oo[r * MID_PITCH] = (uint8_t)finish(acc[r]);
    }
}

// ---- V pass: mid -> S values, handed to an epilogue -------------------------------------
// rows_v: shared-memory copy of the packed rows of block rows 0..FBH-1.
// Epilogue::prefetch(block_row, strip) issues the loads the epilogue will need (feather alpha)
// BEFORE the multiply-adds, Epilogue::row(pre, block_row, strip, s) consumes them.
template <int TAPS, int N, class Epilogue>
__device__ __forceinline__ void vpass(const uint8_t* __restrict__ mid, const int32_t* rows_v, int iy0, Epilogue& epi,
                                      int row_begin, int row_end) {
    constexpr int STRIPS = FBW * 3 / 4;             // 96
    const int total = (row_end - row_begin) * STRIPS;
#pragma unroll 2
    for (int it = threadIdx.x; it < total; it += kT) {
        const int rr = it / STRIPS, strip = it - rr * STRIPS;
        const int r = row_begin + rr;
        const int4* rp = reinterpret_cast<const int4*>(rows_v + r * (TAPS + 1));
        const PackedRow<TAPS> row = read_row<TAPS>([&](int i) { return rp[i]; });
        const uint8_t* m = mid + (size_t)(row.first - iy0) * MID_PITCH + 4 * strip;
        const typename Epilogue::Pre pre = epi.prefetch(r, strip);
        uint32_t w[N];
#pragma unroll
        for (int t = 0; t < N; ++t) w[t] = *reinterpret_cast<const uint32_t*>(m + (size_t)t * MID_PITCH);
        int acc[R];
        dot4<TAPS, N>(w, row, acc);
        uint32_t s[R];
#pragma unroll
        for (int q = 0; q < R; ++q) s[q] = finish(acc[q]);
        epi.row(pre, r, strip, s);
    }
}

// Shared-memory sizing shared by host and device.
__host__ __device__ inline int plane_words(int patch_w) { return patch_w + MAXTAPS + 1; }
__host__ __device__ inline int in_groups(int patch_h) { return (patch_h + 3) / 4; }
__host__ __device__ inline size_t in_bytes(int patch_w, int patch_h) {
    return (size_t)in_groups(patch_h) * 3 * plane_words(patch_w) * 4;
}
__host__ __device__ inline size_t mid_bytes(int patch_h) {
    return ((size_t)((patch_h + 3) / 4 * 4 + 1) * MID_PITCH + 15) / 16 * 16;
}
constexpr size_t kHeadBytes = USDU_JOB_WORDS * 4 + (size_t)FBH * (MAXTAPS + 1) * 4;   // job record + rows_v

}  // namespace fast
}  // namespace usdu
