// usdu_png_decode.cu -- PNGs posted by HTTP workers (static-mode tiles, collector images) -> u8 RGB frames, on the device;
// and the collector master's gather of decoded frames into its fp32 result.
//
// A worker of the reference's protocol posts each processed tile as a PIL PNG at compress_level=0: one IHDR, IDAT
// chunks holding a zlib stream of STORED deflate blocks, and rows filtered per row with None / Sub / Up / Avg / Paeth.
// The master's route handler validates every file on the host (http_master.parse_png) and records, per frame, the
// segments of the uploaded bytes that hold the filtered stream R (per row: the filter byte, then the row's W*C bytes),
// skipping chunk framing, the zlib header and the stored-block headers.  A stream with compressed blocks is inflated on
// the host and its R uploaded as one segment.  What is left on the device is byte moving plus PNG un-filtering, and the
// conversion PIL's convert("RGB") does: grey (C = 1) replicated, grey+alpha (2) and RGBA (4) drop the alpha.
//
// Un-filtering is serial along a row (Sub, Avg, Paeth read the pixel to the left) and down the rows (Up, Avg, Paeth read
// the row above), so one CTA per frame runs a CHUNKED WAVEFRONT: warp w of D owns rows w, w + D, ...; a row is cut into
// chunks of 32 pixels, one pixel per lane; chunk k of row r starts once row r - 1 has published chunk k.  Decoded rows
// live in a shared-memory ring of D rows (warp w's slot), so before a warp overwrites chunk k of its slot it waits
// until the row after the previous occupant has read it (chunk k + 1 too: Paeth's upper-left pixel).  Progress counters
// in shared memory (row * chunks + chunks published) order the warps.  The ring depth D, and with it the warps per CTA,
// is min(16, opt-in shared memory / max_row_bytes): 16 up to 14,524-byte rows (tiles), 3 at 65,536 (16,384 RGBA px).
// Any D >= 2 is deadlock-free: the warp a row waits on (the row above, or the row after its slot's previous occupant)
// only ever waits on rows further up.
//   None, Up  lane-parallel;  Sub  a warp scan per channel, mod 256, carried across chunks;
//   Avg, Paeth  serial per channel inside the chunk (lanes 0..C-1), in place in the ring slot.
#include "usdu_common.cuh"

namespace usdu {
namespace {

constexpr int kDecWarps = 16;                     // the deepest ring; the launch picks D <= kDecWarps warps
constexpr int kDecThreads = kDecWarps * 32;
constexpr int kDecMinWarps = 2;
constexpr int kChunk = 32;                        // pixels per chunk, one per lane

__device__ __forceinline__ int ld_volatile(const int* p) { return *reinterpret_cast<const volatile int*>(p); }

__device__ __forceinline__ void wait_progress(const int* prog, int need) {
    if ((threadIdx.x & 31) == 0)
        while (ld_volatile(prog) < need) {
        }
    __syncwarp();
    __threadfence_block();
}

// The bytes of R from raw position q on: each lane walks its own segment cursor forward (positions only grow per lane).
struct SegCursor {
    const int64_t* segs;    // this frame's segments: (src offset, raw start) pairs
    int n;                  // segments of this frame
    int64_t raw_len;        // |R|
    int s;                  // current segment
    __device__ __forceinline__ uint32_t byte(const uint8_t* src, int64_t q) {
        while (s + 1 < n && segs[2 * (s + 1) + 1] <= q) ++s;
        return src[segs[2 * s] + (q - segs[2 * s + 1])];
    }
};

__device__ __forceinline__ uint32_t paeth(uint32_t a, uint32_t b, uint32_t c) {
    const int p = (int)a + (int)b - (int)c;
    const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__global__ void __launch_bounds__(kDecThreads) png_decode_kernel(const uint8_t* __restrict__ src,
                                                                 const int64_t* __restrict__ segs, int64_t n_segs,
                                                                 const int64_t* __restrict__ descs,
                                                                 uint8_t* __restrict__ dst) {
    extern __shared__ __align__(16) uint8_t ring[];
    __shared__ int prog[kDecWarps];
    const int64_t* d = descs + (int64_t)blockIdx.x * USDU_PNG_DESC_WORDS;
    const int64_t seg0 = d[0], nseg = d[1];
    const int H = (int)d[2], W = (int)d[3], C = (int)d[4];
    uint8_t* out = dst + d[5];
    if (seg0 < 0 || nseg < 1 || seg0 + nseg > n_segs) return;          // the launcher checked the host tables
    const int n = W * C;                                                // bytes of a decoded row
    const int nch = (W + kChunk - 1) / kChunk;
    const int D = blockDim.x >> 5;                                      // ring depth = warps
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < D) prog[threadIdx.x] = 0;
    __syncthreads();

    SegCursor cur{segs + 2 * seg0, (int)nseg, (int64_t)H * (n + 1), 0};
    uint8_t* mine = ring + warp * n;
    for (int r = warp; r < H; r += D) {
        const uint8_t* above = r > 0 ? ring + ((r - 1) % D) * n : nullptr;
        const int* prog_above = &prog[(r - 1 + D) % D];
        const int* prog_next = &prog[(warp + 1) % D];                   // the row after this slot's previous occupant
        const int64_t row_raw = (int64_t)r * (n + 1);
        const uint32_t filt = __shfl_sync(0xffffffffu, lane == 0 ? cur.byte(src, row_raw) : 0u, 0);
        uint32_t carry[4] = {0, 0, 0, 0};                               // Sub: last decoded pixel of the previous chunk
        for (int k = 0; k < nch; ++k) {
            const int x = k * kChunk + lane;
            const int cnt = min(kChunk, W - k * kChunk);
            // the slot's previous occupant (row r - D) must have been read up to chunk k + 1 by row r - D + 1
            if (r >= D) wait_progress(prog_next, (r - D + 1) * nch + min(k + 2, nch));
            if (r > 0 && (filt >= 2)) wait_progress(prog_above, (r - 1) * nch + k + 1);
            uint32_t v[4] = {0, 0, 0, 0};
            if (lane < cnt) {
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c < C) v[c] = cur.byte(src, row_raw + 1 + (int64_t)x * C + c);
            }
            if (filt == 1) {                                            // Sub: inclusive scan over the chunk, per channel
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    uint32_t s = v[c];
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
                        if (lane >= o) s += t;
                    }
                    v[c] = (s + carry[c]) & 0xffu;
                    carry[c] = __shfl_sync(0xffffffffu, v[c], cnt - 1);
                }
            } else if (filt == 2 && lane < cnt && r > 0) {              // Up
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c < C) v[c] = (v[c] + above[x * C + c]) & 0xffu;
            }
            if (lane < cnt) {
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c < C) mine[x * C + c] = (uint8_t)v[c];
            }
            __syncwarp();
            if (filt >= 3 && lane < C) {                                // Avg, Paeth: serial per channel, in place
                const int c = lane;
                uint32_t left = k > 0 ? mine[(k * kChunk - 1) * C + c] : 0u;
                uint32_t ul = (k > 0 && r > 0) ? above[(k * kChunk - 1) * C + c] : 0u;
                for (int i = 0; i < cnt; ++i) {
                    const int o = (k * kChunk + i) * C + c;
                    const uint32_t up = r > 0 ? above[o] : 0u;
                    const uint32_t f = mine[o];
                    const uint32_t pred = filt == 3 ? ((left + up) >> 1) : paeth(left, up, ul);
                    left = (f + pred) & 0xffu;
                    mine[o] = (uint8_t)left;
                    ul = up;
                }
            }
            __syncwarp();
            if (lane < cnt) {                                           // convert("RGB") and store
                const uint8_t* p = mine + x * C;
                uint8_t* q = out + ((int64_t)r * W + x) * 3;
                const uint8_t c0 = p[0];
                q[0] = c0;
                q[1] = C >= 3 ? p[1] : c0;
                q[2] = C >= 3 ? p[2] : c0;
            }
            __threadfence_block();
            __syncwarp();
            if (lane == 0) *reinterpret_cast<volatile int*>(&prog[warp]) = r * nch + k + 1;
        }
    }
}

// The general entry: a PNG of any colour type and bit depth, interlaced or not, its filtered stream R inflated on the
// host (http_master.parse_png_general) and uploaded whole.  One CTA per (frame, pass): a non-interlaced frame is one
// pass; Adam7's seven passes are independent PNG sub-images that scatter to (y0 + i*dy, x0 + j*dx).  The same chunked
// wavefront, on PNG filter units of bpp = max(1, depth*C/8) bytes: a lane owns one unit (a pixel at depth >= 8, one
// byte of 8/depth pixels below), a chunk is 32 units.  The store step converts as PIL's convert("RGB"): sub-byte grey
// scaled to 0..255, 16-bit grey clipped to 255 (PIL's I;16), other 16-bit samples by their high byte, palette indices
// looked up in a 256-entry table (entries past the PLTE's are zero), alpha dropped.
__global__ void __launch_bounds__(kDecThreads) png_decode_general_kernel(const uint8_t* __restrict__ src,
                                                                         const int64_t* __restrict__ descs,
                                                                         uint8_t* __restrict__ dst) {
    extern __shared__ __align__(16) uint8_t ring[];
    __shared__ int prog[kDecWarps];
    const int64_t* d = descs + (int64_t)blockIdx.x * USDU_PNG_GENERAL_DESC_WORDS;
    const uint8_t* R = src + d[0];
    const int W = (int)d[1], H = (int)d[2];                            // the pass's columns and rows
    const int x0 = (int)d[3], y0 = (int)d[4], dx = (int)d[5], dy = (int)d[6];
    const int64_t pitch = d[7];                                         // the frame's width
    const int color = (int)d[8], depth = (int)d[9];
    uint8_t* out = dst + d[10];
    const uint8_t* pal = src + d[11];
    const int C = color == 2 ? 3 : color == 4 ? 2 : color == 6 ? 4 : 1;
    const int bpp = max(1, depth * C / 8);
    const int n = (int)(((int64_t)W * depth * C + 7) / 8);             // filtered bytes of a row
    const int units = (n + bpp - 1) / bpp;
    const int nch = (units + kChunk - 1) / kChunk;
    const int D = blockDim.x >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < D) prog[threadIdx.x] = 0;
    __syncthreads();

    uint8_t* mine = ring + warp * n;
    for (int r = warp; r < H; r += D) {
        const uint8_t* above = r > 0 ? ring + ((r - 1) % D) * n : nullptr;
        const int* prog_above = &prog[(r - 1 + D) % D];
        const int* prog_next = &prog[(warp + 1) % D];
        const uint8_t* row = R + (int64_t)r * (n + 1);
        const uint32_t filt = __shfl_sync(0xffffffffu, lane == 0 ? (uint32_t)row[0] : 0u, 0);
        uint32_t carry[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int k = 0; k < nch; ++k) {
            const int u = k * kChunk + lane;
            const int cnt = min(kChunk, units - k * kChunk);
            if (r >= D) wait_progress(prog_next, (r - D + 1) * nch + min(k + 2, nch));
            if (r > 0 && (filt >= 2)) wait_progress(prog_above, (r - 1) * nch + k + 1);
            uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (lane < cnt) {
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < bpp) v[c] = row[1 + u * bpp + c];
            }
            if (filt == 1) {                                            // Sub: inclusive scan per unit byte
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    if (c >= bpp) break;                                // bpp is uniform over the warp
                    uint32_t s = v[c];
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
                        if (lane >= o) s += t;
                    }
                    v[c] = (s + carry[c]) & 0xffu;
                    carry[c] = __shfl_sync(0xffffffffu, v[c], cnt - 1);
                }
            } else if (filt == 2 && lane < cnt && r > 0) {              // Up
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < bpp) v[c] = (v[c] + above[u * bpp + c]) & 0xffu;
            }
            if (lane < cnt) {
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < bpp) mine[u * bpp + c] = (uint8_t)v[c];
            }
            __syncwarp();
            if (filt >= 3 && lane < bpp) {                              // Avg, Paeth: serial per unit byte, in place
                const int c = lane;
                uint32_t left = k > 0 ? mine[(k * kChunk - 1) * bpp + c] : 0u;
                uint32_t ul = (k > 0 && r > 0) ? above[(k * kChunk - 1) * bpp + c] : 0u;
                for (int i = 0; i < cnt; ++i) {
                    const int o = (k * kChunk + i) * bpp + c;
                    const uint32_t up = r > 0 ? above[o] : 0u;
                    const uint32_t f = mine[o];
                    const uint32_t pred = filt == 3 ? ((left + up) >> 1) : paeth(left, up, ul);
                    left = (f + pred) & 0xffu;
                    mine[o] = (uint8_t)left;
                    ul = up;
                }
            }
            __syncwarp();
            if (lane < cnt) {                                           // convert("RGB") and store
                uint8_t* q = out + ((int64_t)(y0 + r * dy) * pitch + x0) * 3;
                if (depth >= 8) {
                    const uint8_t* p = mine + u * bpp;
                    const int s = depth >> 3;                           // bytes per sample
                    uint32_t c0, c1, c2;
                    if (color == 3) {
                        c0 = pal[3 * p[0]], c1 = pal[3 * p[0] + 1], c2 = pal[3 * p[0] + 2];
                    } else if (color == 2 || color == 6) {
                        c0 = p[0], c1 = p[s], c2 = p[2 * s];
                    } else if (color == 0 && depth == 16) {
                        c0 = c1 = c2 = min(((uint32_t)p[0] << 8) | p[1], 255u);
                    } else {
                        c0 = c1 = c2 = p[0];
                    }
                    uint8_t* o = q + (int64_t)u * dx * 3;
                    o[0] = (uint8_t)c0, o[1] = (uint8_t)c1, o[2] = (uint8_t)c2;
                } else {                                                // 8 / depth pixels in this byte
                    const uint32_t b = mine[u];
                    const int per = 8 / depth, mask = (1 << depth) - 1, scale = 255 / mask;
                    for (int i = 0; i < per; ++i) {
                        const int x = u * per + i;
                        if (x >= W) break;                              // the row's padding bits
                        const uint32_t sv = (b >> (8 - depth * (i + 1))) & mask;
                        uint8_t* o = q + (int64_t)x * dx * 3;
                        if (color == 3) {
                            o[0] = pal[3 * sv], o[1] = pal[3 * sv + 1], o[2] = pal[3 * sv + 2];
                        } else {
                            o[0] = o[1] = o[2] = (uint8_t)(sv * scale);
                        }
                    }
                }
            }
            __threadfence_block();
            __syncwarp();
            if (lane == 0) *reinterpret_cast<volatile int*>(&prog[warp]) = r * nch + k + 1;
        }
    }
}

// frame i of n: dst[i * frame_elems + e] = frames[i][e] / 255 (dequant_u8_fast, bit-identical to __fdiv_rn).  Each
// thread writes 4 consecutive floats with one 16-byte store, from the frame's first 16-byte-aligned output element on
// (its `head` elements before that are written singly), so a dst in mapped host memory gets whole 128-byte lines.
__global__ void __launch_bounds__(kThreads) gather_unpack_kernel(const uint8_t* const* __restrict__ frames, int n,
                                                                 int64_t frame_elems, float* __restrict__ dst) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int f = blockIdx.y; f < n; f += gridDim.y) {
        const uint8_t* src = frames[f];
        float* out = dst + (int64_t)f * frame_elems;
        const int64_t lead = (int64_t)(((16u - ((uintptr_t)out & 15u)) & 15u) >> 2);
        const int64_t head = lead < frame_elems ? lead : frame_elems;
        const int64_t groups = (frame_elems - head) >> 2;
        if (tid < head) out[tid] = dequant_u8_fast(src[tid]);
        const uint8_t* s = src + head;
        float4* o4 = reinterpret_cast<float4*>(out + head);
        for (int64_t g = tid; g < groups; g += stride) {
            const uint8_t* p = s + 4 * g;                               // any alignment: four byte loads
            o4[g] = make_float4(dequant_u8_fast(p[0]), dequant_u8_fast(p[1]), dequant_u8_fast(p[2]),
                                dequant_u8_fast(p[3]));
        }
        const int64_t tail = head + 4 * groups;
        if (tid < frame_elems - tail) out[tail + tid] = dequant_u8_fast(s[4 * groups + tid]);
    }
}

int decode_warps(const void* kernel, const char* what, int max_row_bytes, int* warps) {
    USDU_REQUIRE(max_row_bytes >= 1 && max_row_bytes <= USDU_PNG_MAX_ROW_BYTES,
                 "%s: row bytes %d outside [1, %d]", what, max_row_bytes, USDU_PNG_MAX_ROW_BYTES);
    int dev = 0, optin = 0;
    USDU_CUDA(cudaGetDevice(&dev));
    USDU_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaFuncAttributes a;
    USDU_CUDA(cudaFuncGetAttributes(&a, kernel));
    const int64_t fit = ((int64_t)optin - (int64_t)a.sharedSizeBytes) / max_row_bytes;
    USDU_REQUIRE(fit >= kDecMinWarps, "%s: %d-byte rows leave room for %lld ring rows (need %d)", what,
                 max_row_bytes, (long long)fit, kDecMinWarps);
    *warps = fit < kDecWarps ? (int)fit : kDecWarps;
    return USDU_OK;
}

}  // namespace
}  // namespace usdu

using namespace usdu;

extern "C" {

int usdu_png_decode_warps(int max_row_bytes) {
    int warps = 0;
    const int r = decode_warps((const void*)png_decode_kernel, "usdu_png_decode_u8", max_row_bytes, &warps);
    return r != USDU_OK ? r : warps;
}

int usdu_png_decode_u8(const uint8_t* src_dev, const int64_t* segs_dev, int64_t n_segs, const int64_t* descs_dev,
                       int n, int max_row_bytes, uint8_t* dst_dev, void* stream) {
    USDU_REQUIRE(n >= 0, "usdu_png_decode_u8: %d frames", n);
    if (n == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && segs_dev && descs_dev && dst_dev, "usdu_png_decode_u8: null pointer");
    USDU_REQUIRE(n_segs >= 1, "usdu_png_decode_u8: no segments");
    int warps = 0;
    int r = decode_warps((const void*)png_decode_kernel, "usdu_png_decode_u8", max_row_bytes, &warps);
    if (r != USDU_OK) return r;
    const size_t smem = (size_t)warps * (size_t)max_row_bytes;
    r = raise_smem_limit((const void*)png_decode_kernel, smem);
    if (r != USDU_OK) return r;
    png_decode_kernel<<<n, warps * 32, smem, (cudaStream_t)stream>>>(src_dev, segs_dev, n_segs, descs_dev, dst_dev);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_png_decode_general_u8(const uint8_t* src_dev, const int64_t* descs_dev, int n, int max_row_bytes,
                               uint8_t* dst_dev, void* stream) {
    USDU_REQUIRE(n >= 0, "usdu_png_decode_general_u8: %d passes", n);
    if (n == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && descs_dev && dst_dev, "usdu_png_decode_general_u8: null pointer");
    int warps = 0;
    int r = decode_warps((const void*)png_decode_general_kernel, "usdu_png_decode_general_u8", max_row_bytes, &warps);
    if (r != USDU_OK) return r;
    const size_t smem = (size_t)warps * (size_t)max_row_bytes;
    r = raise_smem_limit((const void*)png_decode_general_kernel, smem);
    if (r != USDU_OK) return r;
    png_decode_general_kernel<<<n, warps * 32, smem, (cudaStream_t)stream>>>(src_dev, descs_dev, dst_dev);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_gather_unpack_f32(const uint8_t* const* frames_dev, int n, int64_t frame_elems, float* dst, void* stream) {
    USDU_REQUIRE(n >= 0 && frame_elems >= 0, "usdu_gather_unpack_f32: %d frames of %lld elements", n,
                 (long long)frame_elems);
    if (n == 0 || frame_elems == 0) return USDU_OK;
    USDU_REQUIRE(frames_dev && dst, "usdu_gather_unpack_f32: null pointer");
    USDU_REQUIRE(((uintptr_t)dst & 3) == 0, "usdu_gather_unpack_f32: dst must be 4-byte aligned");
    // pinned host memory is written through its device alias (the same address under UVA, cudaHostAlloc)
    cudaPointerAttributes pa;
    USDU_CUDA(cudaPointerGetAttributes(&pa, dst));
    float* out = dst;
    if (pa.type == cudaMemoryTypeHost) {
        void* alias = nullptr;
        USDU_CUDA(cudaHostGetDevicePointer(&alias, dst, 0));
        out = static_cast<float*>(alias);
    } else {
        USDU_REQUIRE(pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged,
                     "usdu_gather_unpack_f32: dst is neither device nor pinned host memory");
    }
    const int64_t groups = frame_elems / 4 + 1;
    const int gy = min(n, 65535);
    const int want = max(1, 4 * grid_sms() / gy);                       // about 4 CTAs per SM over the whole grid
    const int64_t need = (groups + kThreads - 1) / kThreads;
    const int gx = need < want ? (int)need : want;
    gather_unpack_kernel<<<dim3(gx, gy), kThreads, 0, (cudaStream_t)stream>>>(frames_dev, n, frame_elems, out);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

}  // extern "C"
