// usdu_png.cu -- u8 frames -> PNG files on the device: base64 text of a stored (deflate level 0, filter "None") PNG for
// the collector worker, and Pillow's level-0 PNG, filters and all, for the HTTP tile worker (the second half of the file).
//
// The reference's collector worker sends every image as base64 of a PIL PNG at compress_level=0
// (nodes/collector.py:84-119).  At level 0 the deflate blocks are stored, so a PNG is layout plus two checksums:
// CRC-32 per chunk and Adler-32 over the raw stream R (per row: filter byte 0, then the row's W*C bytes).  The
// layout the kernels write, byte for byte (include/usdu_b200.h, usdu_png_base64_u8; tests/png_model.py):
//   signature | IHDR | IDAT k = [78 01 if k == 0] + stored block k of R | IDAT(Adler-32 of R) | IEND
// Block k holds R[k*65535, ...) (the last one shorter), alone in chunk k, so every chunk offset is known on the host
// and the Adler trailer's own chunk keeps every other chunk's CRC independent of it.
//
//   Pass A  png_idat_kernel      one CTA per (frame, block): gathers the block's rows into shared memory with the
//                                filter bytes and the chunk / stored-block headers, computes the chunk's CRC and the
//                                block's Adler partials, writes the chunk.
//   Pass B  png_frame_kernel     one CTA per frame: combines the Adler partials, writes signature, IHDR, the Adler
//                                chunk and IEND.
//   Pass C  png_base64_kernel    3 bytes in, 4 characters out; each thread 12 bytes -> 16 characters.
//
// CRC in parallel: with raw(x) the table CRC from a zero register and no final inversion, raw(A || B) =
// raw(A) * x^(8|B|) ^ raw(B) (mod P), leading zero bytes leave raw unchanged, and the standard CRC-32 of a
// message is ~raw of the message with its first 4 bytes inverted.  The chunk body (type + data) is right-aligned in a
// zero-padded shared buffer of kPngThreads fixed-size segments; each thread CRCs one segment and the segments combine
// with the compile-time multipliers x^(8 * kSeg * 2^j).
//
// Pillow's level-0 PNG (usdu_png_encode_u8) has a framing the host reads off Pillow for the shape (http_worker.png_layout),
// so the kernels only fill it in:
//   Pass 1  png_filter_kernel       one warp per row: Pillow's filter choice, the filtered row into R (scratch), the
//                                   row's Adler partials.
//   Pass 2  png_adler_frame_kernel  one CTA per frame: the Adler-32 of R, the template bytes outside the IDAT chunks.
//   Pass 3  png_chunk_kernel        one CTA per (IDAT chunk, frame): template + R + Adler bytes spliced in shared
//                                   memory, the chunk's CRC as above, the chunk written.
#include "usdu_common.cuh"

namespace usdu {
namespace {

constexpr int kPngThreads = 256;
constexpr uint32_t kStored = 65535;                      // bytes of R per stored deflate block
constexpr uint32_t kSeg = 260;                           // CRC segment per thread, bytes (a multiple of 4)
constexpr uint32_t kSpan = kPngThreads * kSeg;           // >= 4 (type) + 2 (zlib header) + 5 (block header) + 65535
constexpr uint32_t kCrcPoly = 0xEDB88320u;               // reflected CRC-32
constexpr uint32_t kAdlerMod = 65521u;
constexpr int64_t kChunkStride = 12 + 5 + kStored;       // bytes of a full block's chunk (chunk 0 has 2 more)
constexpr int64_t kFirstChunk = 8 + 25;                  // signature + IHDR chunk
static_assert(kSpan >= 4 + 2 + 5 + kStored, "CRC span too short for one chunk body");
static_assert(kSeg % 4 == 0, "segments are read as words");

// x^(8 * nbytes) mod P in the reflected representation (bit 31 = x^0), at compile time.
constexpr uint32_t xpow8(uint32_t nbytes) {
    uint32_t v = 0x80000000u;
    for (uint64_t i = 0; i < 8ull * nbytes; ++i) v = (v >> 1) ^ ((v & 1u) ? kCrcPoly : 0u);
    return v;
}
constexpr uint32_t kShift1 = xpow8(kSeg), kShift2 = xpow8(2 * kSeg), kShift4 = xpow8(4 * kSeg);
constexpr uint32_t kShift8 = xpow8(8 * kSeg), kShift16 = xpow8(16 * kSeg), kShift32 = xpow8(32 * kSeg);

// a * b mod P, reflected (zlib's multmodp with a fixed trip count)
__device__ __forceinline__ uint32_t gf_mul(uint32_t a, uint32_t b) {
    uint32_t p = 0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b >> 1) ^ ((b & 1u) ? kCrcPoly : 0u);
    }
    return p;
}

// x^(8 * kSpan): moves a raw CRC past one whole span (the filtered encoder's chunks may take several)
constexpr uint32_t gf_mul_c(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; ++i) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b >> 1) ^ ((b & 1u) ? kCrcPoly : 0u);
    }
    return p;
}
constexpr uint32_t kShift64 = gf_mul_c(kShift32, kShift32), kShift128 = gf_mul_c(kShift64, kShift64);
constexpr uint32_t kShiftSpan = gf_mul_c(kShift128, kShift128);

__device__ __forceinline__ void crc_table_init(uint32_t* table, int tid) {
    for (int t = tid; t < 256; t += kPngThreads) {
        uint32_t c = t;
        for (int j = 0; j < 8; ++j) c = (c >> 1) ^ ((c & 1u) ? kCrcPoly : 0u);
        table[t] = c;
    }
}

// Raw CRC of the kSpan-byte shared buffer whose first s0 bytes are zero: each thread CRCs its kSeg-byte segment and the
// segments combine in the warp; lane 0 returns its warp's raw CRC (span_crc_combine joins the warps).
__device__ __forceinline__ uint32_t span_crc_warp(const uint32_t* body_words, const uint32_t* table, int tid,
                                                  uint32_t s0) {
    // segment i is followed by (kPngThreads - 1 - i) * kSeg bytes
    uint32_t crc = 0;
    if ((uint32_t)(tid + 1) * kSeg > s0) {
        const uint32_t* seg = body_words + tid * (kSeg / 4);
#pragma unroll 4
        for (uint32_t i = 0; i < kSeg / 4; ++i) {
            crc ^= seg[i];
            crc = table[crc & 0xff] ^ (crc >> 8);
            crc = table[crc & 0xff] ^ (crc >> 8);
            crc = table[crc & 0xff] ^ (crc >> 8);
            crc = table[crc & 0xff] ^ (crc >> 8);
        }
    }
    crc = gf_mul(kShift1, crc) ^ __shfl_down_sync(0xffffffffu, crc, 1);
    crc = gf_mul(kShift2, crc) ^ __shfl_down_sync(0xffffffffu, crc, 2);
    crc = gf_mul(kShift4, crc) ^ __shfl_down_sync(0xffffffffu, crc, 4);
    crc = gf_mul(kShift8, crc) ^ __shfl_down_sync(0xffffffffu, crc, 8);
    crc = gf_mul(kShift16, crc) ^ __shfl_down_sync(0xffffffffu, crc, 16);
    return crc;
}

__device__ __forceinline__ uint32_t span_crc_combine(const uint32_t* warp_crc) {
    uint32_t c = 0;
    for (int w = 0; w < kPngThreads / 32; ++w) c = gf_mul(kShift32, c) ^ warp_crc[w];
    return c;
}

// m bytes of the shared buffer from byte src0 on to global g, with aligned word stores where g allows
__device__ __forceinline__ void copy_out(uint8_t* g, const uint32_t* body_words, uint32_t src0, uint32_t m, int tid) {
    const uint8_t* body = reinterpret_cast<const uint8_t*>(body_words);
    uint32_t head = (4u - (uint32_t)((uintptr_t)g & 3)) & 3u;
    head = head < m ? head : m;
    const uint32_t nw = (m - head) / 4;
    for (uint32_t i = tid; i < head; i += kPngThreads) g[i] = body[src0 + i];
    {
        const uint32_t so = src0 + head;
        const uint32_t sh = (so & 3u) * 8u;
        const uint32_t* sw = body_words + (so >> 2);
        uint32_t* gw = reinterpret_cast<uint32_t*>(g + head);
        for (uint32_t i = tid; i < nw; i += kPngThreads) gw[i] = __funnelshift_r(sw[i], sw[i + 1], sh);
    }
    for (uint32_t i = head + 4 * nw + tid; i < m; i += kPngThreads) g[i] = body[src0 + i];
}

__device__ __forceinline__ uint32_t crc_bitwise(uint32_t c, const uint8_t* p, int n) {
    for (int i = 0; i < n; ++i) {
        c ^= p[i];
        for (int j = 0; j < 8; ++j) c = (c >> 1) ^ ((c & 1u) ? kCrcPoly : 0u);
    }
    return c;
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    return v;
}

struct PngGeom {
    int64_t row_bytes;   // W * C
    int64_t rowlen;      // 1 + W * C
    int64_t raw;         // |R| = H * rowlen
    int64_t nblk;        // stored blocks
    int64_t png_len;
    int64_t text_len;
    int64_t png_area;    // png_len rounded up to 48: the staging bytes pass C reads
    int64_t stride;      // staging bytes per frame: png_area + 16 * nblk (Adler partials)
};

int png_geom(int H, int W, int C, PngGeom* g) {
    USDU_REQUIRE(C >= 2 && C <= 4, "usdu_png: %d channels: a PNG frame has 2 (LA), 3 (RGB) or 4 (RGBA)", C);
    USDU_REQUIRE(H >= 1 && W >= 1, "usdu_png: empty frame %dx%d", W, H);
    g->row_bytes = (int64_t)W * C;
    g->rowlen = g->row_bytes + 1;
    g->raw = (int64_t)H * g->rowlen;
    USDU_REQUIRE(g->raw < ((int64_t)1 << 40), "usdu_png: frame too large");
    g->nblk = (g->raw + kStored - 1) / kStored;
    g->png_len = 63 + 17 * g->nblk + g->raw;
    g->text_len = 4 * ((g->png_len + 2) / 3);
    g->png_area = (g->png_len + 47) / 48 * 48;
    g->stride = g->png_area + 16 * g->nblk;
    return USDU_OK;
}

__host__ __device__ __forceinline__ int64_t chunk_offset(int64_t k) {
    return kFirstChunk + k * kChunkStride + (k > 0 ? 2 : 0);
}

__global__ void __launch_bounds__(kPngThreads)
png_idat_kernel(const uint8_t* __restrict__ src, int64_t frame_bytes, uint32_t row_bytes, uint32_t rowlen, int64_t raw,
                int nblk, uint8_t* __restrict__ staging, int64_t stride, int64_t png_area) {
    extern __shared__ uint32_t body_words[];              // kSpan bytes + one word of slack
    __shared__ uint32_t table[256];
    __shared__ uint32_t warp_crc[kPngThreads / 32];
    __shared__ unsigned long long warp_s1[kPngThreads / 32], warp_s2[kPngThreads / 32];
    uint8_t* body = reinterpret_cast<uint8_t*>(body_words);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k = blockIdx.x, b = blockIdx.y;
    const int64_t a = (int64_t)k * kStored;                // first byte of R in this block
    const uint32_t L = (uint32_t)(raw - a < kStored ? raw - a : kStored);
    const uint32_t hdr = (k == 0 ? 2u : 0u) + 5u;
    const uint32_t n = 4 + hdr + L;                       // CRC'd bytes: chunk type + data
    const uint32_t s0 = kSpan - n;                        // the body is right-aligned; zeros before it

    crc_table_init(table, tid);
    for (uint32_t w = tid; w < (s0 + 3) / 4; w += kPngThreads) body_words[w] = 0;
    if (tid == 0) body_words[kSpan / 4] = 0;              // slack word the funnel-shift copy may read
    __syncthreads();
    if (tid == 0) {
        uint8_t* p = body + s0;
        // the type bytes go in inverted: the CRC register's initial ~0 (see the top of the file)
        p[0] = (uint8_t)~'I'; p[1] = (uint8_t)~'D'; p[2] = (uint8_t)~'A'; p[3] = (uint8_t)~'T';
        p += 4;
        if (k == 0) { *p++ = 0x78; *p++ = 0x01; }          // zlib header: deflate, 32K window, FCHECK
        *p++ = (k == nblk - 1) ? 1 : 0;                    // BFINAL, BTYPE = 00 (stored)
        p[0] = (uint8_t)L; p[1] = (uint8_t)(L >> 8); p[2] = (uint8_t)~L; p[3] = (uint8_t)(~L >> 8);
    }

    // the block's bytes of R: row r, column c (c == 0: the filter byte) <- frame byte r * W * C + c - 1
    const uint8_t* img = src + (int64_t)b * frame_bytes;
    uint8_t* dst = body + s0 + 4 + hdr;
    unsigned long long s1 = 0, s2 = 0;
    {
        const int64_t q = a + tid;
        uint32_t row = (uint32_t)(q / rowlen);
        uint32_t col = (uint32_t)(q - (int64_t)row * rowlen);
        for (uint32_t p = tid; p < L; p += kPngThreads) {
            const uint32_t d = col == 0 ? 0u : (uint32_t)__ldg(img + (int64_t)row * row_bytes + col - 1);
            dst[p] = (uint8_t)d;
            s1 += d;
            s2 += (L - p) * d;                             // < 2^24
            col += kPngThreads;
            if (col >= rowlen) {
                const uint32_t t = col / rowlen;
                row += t;
                col -= t * rowlen;
            }
        }
    }
    __syncthreads();

    const uint32_t crc = span_crc_warp(body_words, table, tid, s0);
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) {
        warp_crc[warp] = crc;
        warp_s1[warp] = s1;
        warp_s2[warp] = s2;
    }

    // copy the chunk data (smem body bytes 4.., n - 4 of them) out with aligned word stores
    uint8_t* frame = staging + (int64_t)b * stride;
    uint8_t* g = frame + chunk_offset(k) + 8;
    const uint32_t m = n - 4, src0 = s0 + 4;
    copy_out(g, body_words, src0, m, tid);
    __syncthreads();

    if (tid == 0) {
        const uint32_t c = span_crc_combine(warp_crc);
        unsigned long long t1 = 0, t2 = 0;
        for (int w = 0; w < kPngThreads / 32; ++w) {
            t1 += warp_s1[w];
            t2 += warp_s2[w];
        }
        uint8_t* chunk = frame + chunk_offset(k);
        put_be32(chunk, m);
        chunk[4] = 'I'; chunk[5] = 'D'; chunk[6] = 'A'; chunk[7] = 'T';
        put_be32(chunk + 8 + m, ~c);
        unsigned long long* part = reinterpret_cast<unsigned long long*>(frame + png_area) + 2 * k;
        part[0] = t1 % kAdlerMod;
        part[1] = t2 % kAdlerMod;
    }
}

__global__ void __launch_bounds__(kPngThreads)
png_frame_kernel(int H, int W, int C, int64_t raw, int nblk, uint8_t* __restrict__ staging, int64_t stride,
                 int64_t png_len, int64_t png_area) {
    __shared__ unsigned long long red1[kPngThreads / 32], red2[kPngThreads / 32];
    const int tid = threadIdx.x;
    uint8_t* frame = staging + (int64_t)blockIdx.x * stride;
    const unsigned long long* part = reinterpret_cast<const unsigned long long*>(frame + png_area);
    // Adler-32 of R from the block partials: s1_k = sum d, s2_k = sum (L_k - j) d_j over block k (both mod 65521);
    // B = |R| + sum_k [s2_k + (|R| - a_k - L_k) s1_k], A = 1 + sum_k s1_k (mod 65521)
    unsigned long long A = 0, Bs = 0;
    for (int k = tid; k < nblk; k += kPngThreads) {
        const int64_t a = (int64_t)k * kStored;
        const int64_t L = raw - a < kStored ? raw - a : kStored;
        const unsigned long long after = (unsigned long long)(raw - a - L) % kAdlerMod;
        A = (A + part[2 * k]) % kAdlerMod;
        Bs = (Bs + part[2 * k + 1] + after * part[2 * k]) % kAdlerMod;
    }
    A = warp_sum(A);
    Bs = warp_sum(Bs);
    if ((tid & 31) == 0) {
        red1[tid >> 5] = A;
        red2[tid >> 5] = Bs;
    }
    __syncthreads();
    if (tid != 0) return;
    for (int w = 1; w < kPngThreads / 32; ++w) {
        A += red1[w];
        Bs += red2[w];
    }
    const uint32_t s1 = (uint32_t)((1 + A) % kAdlerMod);
    const uint32_t s2 = (uint32_t)(((unsigned long long)raw % kAdlerMod + Bs) % kAdlerMod);

    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    for (int i = 0; i < 8; ++i) frame[i] = sig[i];
    uint8_t* ih = frame + 8;
    const uint8_t ctype = C == 2 ? 4 : (C == 3 ? 2 : 6);  // LA, RGB, RGBA: Image.fromarray's modes
    put_be32(ih, 13);
    ih[4] = 'I'; ih[5] = 'H'; ih[6] = 'D'; ih[7] = 'R';
    put_be32(ih + 8, (uint32_t)W);
    put_be32(ih + 12, (uint32_t)H);
    ih[16] = 8; ih[17] = ctype; ih[18] = 0; ih[19] = 0; ih[20] = 0;
    put_be32(ih + 21, ~crc_bitwise(0xffffffffu, ih + 4, 17));

    uint8_t* ad = frame + kFirstChunk + 2 + 17 * (int64_t)nblk + raw;   // after the last (short) block's chunk
    put_be32(ad, 4);
    ad[4] = 'I'; ad[5] = 'D'; ad[6] = 'A'; ad[7] = 'T';
    put_be32(ad + 8, (s2 << 16) | s1);
    put_be32(ad + 12, ~crc_bitwise(0xffffffffu, ad + 4, 8));
    uint8_t* end = ad + 16;
    const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
    for (int i = 0; i < 12; ++i) end[i] = iend[i];
    for (int64_t i = png_len; i < (png_len + 2) / 3 * 3; ++i) frame[i] = 0;   // the last 3-byte group's padding
}

__device__ __forceinline__ uint32_t b64_char(uint32_t v) {
    uint32_t c = v + 'A';
    c += v >= 26 ? 6u : 0u;             // 'a'..'z'
    c -= v >= 52 ? 75u : 0u;            // '0'..'9'
    c -= v >= 62 ? 15u : 0u;            // '+'
    c += v >= 63 ? 3u : 0u;             // '/'
    return c;
}

__device__ __forceinline__ uint32_t b64_group(uint32_t x, uint32_t y, uint32_t z) {
    const uint32_t v = (x << 16) | (y << 8) | z;
    return b64_char(v >> 18) | (b64_char((v >> 12) & 63) << 8) | (b64_char((v >> 6) & 63) << 16) |
           (b64_char(v & 63) << 24);
}

__global__ void __launch_bounds__(kPngThreads)
png_base64_kernel(const uint8_t* __restrict__ staging, int64_t stride, int64_t png_len, int64_t units, int64_t total,
                  char* __restrict__ text, int64_t text_len) {
    const int64_t groups = (png_len + 2) / 3;
    const int rem = (int)(png_len - 3 * (groups - 1));    // 1..3 bytes in the last group
    const int64_t step = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
        const int64_t b = i / units, j = i - b * units;
        const uint32_t* s = reinterpret_cast<const uint32_t*>(staging + b * stride + 12 * j);
        const uint32_t w0 = __ldcs(s), w1 = __ldcs(s + 1), w2 = __ldcs(s + 2);
        uint32_t out[4];
        out[0] = b64_group(w0 & 0xff, (w0 >> 8) & 0xff, (w0 >> 16) & 0xff);
        out[1] = b64_group(w0 >> 24, w1 & 0xff, (w1 >> 8) & 0xff);
        out[2] = b64_group((w1 >> 16) & 0xff, w1 >> 24, w2 & 0xff);
        out[3] = b64_group((w2 >> 8) & 0xff, (w2 >> 16) & 0xff, w2 >> 24);
        uint32_t* o = reinterpret_cast<uint32_t*>(text + b * text_len) + 4 * j;
        const int64_t g0 = 4 * j;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const int64_t g = g0 + m;
            if (g >= groups) break;
            uint32_t v = out[m];
            if (g == groups - 1 && rem < 3) v = rem == 1 ? (v & 0xffffu) | 0x3d3d0000u : (v & 0xffffffu) | 0x3d000000u;
            o[m] = v;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Pillow's level-0 PNG of an RGB frame (usdu_png_encode_u8): the filtered stream R spliced into a framing the host
// derived from Pillow for this shape.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kRowsPerCta = kPngThreads / 32;

__device__ __forceinline__ uint32_t filter_cost(uint32_t v) {
    v &= 0xffu;
    return v < 128u ? v : 256u - v;
}

__device__ __forceinline__ uint32_t paeth_pred(uint32_t a, uint32_t b, uint32_t c) {
    const int p = (int)a + (int)b - (int)c;
    const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// Pass 1, one warp per row: the four filter sums in one sweep over the row and the raw row above, Pillow's choice, then
// the filter byte and the filtered row to R[row * rowlen, ...) in the frame's scratch, and the row's Adler partials
// (s1 = sum d, s2 = sum (rowlen - j) d_j, both mod 65521) to the frame's partial table.
__global__ void __launch_bounds__(kPngThreads)
png_filter_kernel(const uint8_t* __restrict__ src, int H, uint32_t row_bytes, uint8_t* __restrict__ scratch,
                  int64_t stride, int64_t parts_at) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5);
    if (row >= H) return;
    const int b = blockIdx.y;
    const uint8_t* cur = src + ((int64_t)b * H + row) * row_bytes;
    const uint8_t* prev = cur - row_bytes;
    const bool top = row == 0;
    uint32_t s_none = 0, s_up = 0, s_sub = 0, s_paeth = 0;
    for (uint32_t i = lane; i < row_bytes; i += 32) {
        const uint32_t x = __ldg(cur + i);
        const uint32_t a = i >= 3 ? __ldg(cur + i - 3) : 0u;
        const uint32_t u = top ? 0u : __ldg(prev + i);
        const uint32_t c = (top || i < 3) ? 0u : __ldg(prev + i - 3);
        s_none += filter_cost(x);
        s_up += filter_cost(x - u);
        s_sub += filter_cost(x - a);
        s_paeth += filter_cost(x - paeth_pred(a, u, c));
    }
    s_none = __reduce_add_sync(0xffffffffu, s_none);      // < 2^23 for rows of at most USDU_PNG_MAX_ROW_BYTES
    s_up = __reduce_add_sync(0xffffffffu, s_up);
    s_sub = __reduce_add_sync(0xffffffffu, s_sub);
    s_paeth = __reduce_add_sync(0xffffffffu, s_paeth);
    // Pillow tries None, Up, Sub, Paeth in this order and keeps a later one only when its sum is strictly smaller
    uint32_t f = 0, best = s_none;
    if (s_up < best) { f = 2; best = s_up; }
    if (s_sub < best) { f = 1; best = s_sub; }
    if (s_paeth < best) f = 4;

    const uint32_t rowlen = row_bytes + 1;
    uint8_t* frame = scratch + (int64_t)b * stride;
    uint8_t* out = frame + (int64_t)row * rowlen;
    uint32_t s1 = 0;
    unsigned long long s2 = 0;
    for (uint32_t i = lane; i < row_bytes; i += 32) {
        const uint32_t x = __ldg(cur + i);
        uint32_t v = x;
        if (f == 2) {
            v = x - (top ? 0u : __ldg(prev + i));
        } else if (f == 1) {
            v = x - (i >= 3 ? __ldg(cur + i - 3) : 0u);
        } else if (f == 4) {
            const uint32_t a = i >= 3 ? __ldg(cur + i - 3) : 0u;
            const uint32_t u = top ? 0u : __ldg(prev + i);
            const uint32_t c = (top || i < 3) ? 0u : __ldg(prev + i - 3);
            v = x - paeth_pred(a, u, c);
        }
        v &= 0xffu;
        out[1 + i] = (uint8_t)v;
        s1 += v;
        s2 += (unsigned long long)(rowlen - 1 - i) * v;
    }
    if (lane == 0) {
        out[0] = (uint8_t)f;
        s1 += f;
        s2 += (unsigned long long)rowlen * f;
    }
    s1 = __reduce_add_sync(0xffffffffu, s1);               // < 2^25
    s2 = warp_sum(s2);
    if (lane == 0) {
        uint32_t* part = reinterpret_cast<uint32_t*>(frame + parts_at) + 2 * row;
        part[0] = s1 % kAdlerMod;
        part[1] = (uint32_t)(s2 % kAdlerMod);
    }
}

// Pass 2, one CTA per frame: the Adler-32 of R from the row partials (same fold as png_frame_kernel, with a_r = r *
// rowlen and L_r = rowlen) into the frame's scratch word, and the template bytes outside every IDAT chunk (signature,
// IHDR, whatever lies between or after the chunks) into the output.
__global__ void __launch_bounds__(kPngThreads)
png_adler_frame_kernel(int H, uint32_t rowlen, uint8_t* __restrict__ scratch, int64_t stride, int64_t parts_at,
                       const uint8_t* __restrict__ tmpl, int64_t png_len, const int64_t* __restrict__ chunks,
                       int n_chunks, uint8_t* __restrict__ dst) {
    __shared__ unsigned long long red1[kPngThreads / 32], red2[kPngThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x;
    uint8_t* frame = scratch + (int64_t)b * stride;
    const uint32_t* part = reinterpret_cast<const uint32_t*>(frame + parts_at);
    const int64_t raw = (int64_t)H * rowlen;
    unsigned long long A = 0, Bs = 0;
    for (int r = tid; r < H; r += kPngThreads) {
        const unsigned long long after = (unsigned long long)(raw - (int64_t)(r + 1) * rowlen) % kAdlerMod;
        A = (A + part[2 * r]) % kAdlerMod;
        Bs = (Bs + part[2 * r + 1] + after * part[2 * r]) % kAdlerMod;
    }
    A = warp_sum(A);
    Bs = warp_sum(Bs);
    if (lane == 0) {
        red1[warp] = A;
        red2[warp] = Bs;
    }

    uint8_t* out = dst + (int64_t)b * png_len;
    const int64_t head = chunks[0] < png_len ? chunks[0] : png_len;
    for (int64_t i = tid; i < head; i += kPngThreads) out[i] = tmpl[i];
    for (int k = warp; k < n_chunks; k += kPngThreads / 32) {
        const int64_t lo = chunks[2 * k] + 12 + chunks[2 * k + 1];
        int64_t hi = k + 1 < n_chunks ? chunks[2 * k + 2] : png_len;
        hi = hi < png_len ? hi : png_len;
        for (int64_t i = (lo > 0 ? lo : 0) + lane; i < hi; i += 32) out[i] = tmpl[i];
    }
    __syncthreads();
    if (tid != 0) return;
    for (int w = 1; w < kPngThreads / 32; ++w) {
        A += red1[w];
        Bs += red2[w];
    }
    const uint32_t s1 = (uint32_t)((1 + A) % kAdlerMod);
    const uint32_t s2 = (uint32_t)(((unsigned long long)raw % kAdlerMod + Bs) % kAdlerMod);
    *reinterpret_cast<uint32_t*>(frame + parts_at + 8 * (int64_t)H) = (s2 << 16) | s1;
}

struct AdlerAt {
    int64_t p[4];        // file offsets of the Adler-32 bytes, most significant first
};

// Pass 3, one CTA per (IDAT chunk, frame): the chunk's type and data assembled in shared memory -- template bytes, R
// over the runs that fall in the chunk, the Adler bytes that do -- its CRC with the segment-combined scheme, the chunk
// written out.  A chunk longer than one span is done in spans aligned to its end; only the first is zero-padded.
__global__ void __launch_bounds__(kPngThreads)
png_chunk_kernel(const uint8_t* __restrict__ scratch, int64_t stride, int64_t adler_slot, const uint8_t* __restrict__ tmpl,
                 int64_t png_len, const int64_t* __restrict__ runs, int n_runs, const int64_t* __restrict__ chunks,
                 AdlerAt adler_at, uint8_t* __restrict__ dst) {
    extern __shared__ uint32_t body_words[];              // kSpan bytes + one word of slack
    __shared__ uint32_t table[256];
    __shared__ uint32_t warp_crc[kPngThreads / 32];
    __shared__ int first_run;
    uint8_t* body = reinterpret_cast<uint8_t*>(body_words);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k = blockIdx.x, b = blockIdx.y;
    const uint8_t* R = scratch + (int64_t)b * stride;
    const uint32_t adler = *reinterpret_cast<const uint32_t*>(R + adler_slot);
    uint8_t* out = dst + (int64_t)b * png_len;
    const int64_t off = chunks[2 * k], len = chunks[2 * k + 1];
    const int64_t lo0 = off + 4, end = off + 8 + len;     // CRC'd bytes: chunk type + data
    if (off < 0 || len < 0 || end + 4 > png_len) return;  // not a chunk of this file: leave the output alone
    const int64_t nwin = (end - lo0 + kSpan - 1) / kSpan;

    crc_table_init(table, tid);
    uint32_t total = 0;                                   // raw CRC so far (thread 0)
    for (int64_t w = 0; w < nwin; ++w) {
        const int64_t hi = end - (nwin - 1 - w) * (int64_t)kSpan;
        const int64_t lo = hi - kSpan > lo0 ? hi - kSpan : lo0;
        const uint32_t s0 = kSpan - (uint32_t)(hi - lo);  // the bytes are right-aligned; zeros before them
        for (uint32_t i = tid; i < (s0 + 3) / 4; i += kPngThreads) body_words[i] = 0;
        if (tid == 0) {
            body_words[kSpan / 4] = 0;                    // slack word the funnel-shift copy may read
            int l = 0, h = n_runs;                        // first run ending after lo
            while (l < h) {
                const int m = (l + h) >> 1;
                if (runs[3 * m] + runs[3 * m + 2] <= lo) l = m + 1; else h = m;
            }
            first_run = l;
        }
        __syncthreads();
        for (int64_t p = lo + tid; p < hi; p += kPngThreads) body[s0 + (p - lo)] = tmpl[p];
        __syncthreads();
        for (int j = first_run; j < n_runs && runs[3 * j] < hi; ++j) {
            const int64_t f = runs[3 * j], s = runs[3 * j + 1], n = runs[3 * j + 2];
            const int64_t a = f > lo ? f : lo, e = f + n < hi ? f + n : hi;
            for (int64_t p = a + tid; p < e; p += kPngThreads) body[s0 + (p - lo)] = R[s + (p - f)];
        }
        if (tid == 0) {
            for (int i = 0; i < 4; ++i) {
                const int64_t p = adler_at.p[i];
                if (p >= lo && p < hi) body[s0 + (p - lo)] = (uint8_t)(adler >> (24 - 8 * i));
            }
            // the type bytes go in inverted: the CRC register's initial ~0 (see the top of the file); they are not
            // copied out from here
            for (int64_t p = lo0; p < lo0 + 4; ++p)
                if (p >= lo && p < hi) body[s0 + (p - lo)] ^= 0xffu;
        }
        __syncthreads();
        const uint32_t crc = span_crc_warp(body_words, table, tid, s0);
        if (lane == 0) warp_crc[warp] = crc;
        const int64_t d0 = lo > off + 8 ? lo : off + 8;   // chunk data in this span
        if (hi > d0) copy_out(out + d0, body_words, s0 + (uint32_t)(d0 - lo), (uint32_t)(hi - d0), tid);
        __syncthreads();
        if (tid == 0) total = gf_mul(kShiftSpan, total) ^ span_crc_combine(warp_crc);
    }
    if (tid == 0) {
        for (int i = 0; i < 8; ++i) out[off + i] = tmpl[off + i];   // length and type
        put_be32(out + end, ~total);
    }
}

}  // namespace
}  // namespace usdu

using namespace usdu;

extern "C" {

int usdu_png_sizes(int H, int W, int C, int64_t* png_len, int64_t* text_len, int64_t* staging_bytes) {
    USDU_REQUIRE(png_len && text_len && staging_bytes, "usdu_png_sizes: null pointer");
    PngGeom g;
    const int s = png_geom(H, W, C, &g);
    if (s != USDU_OK) return s;
    *png_len = g.png_len;
    *text_len = g.text_len;
    *staging_bytes = g.stride;
    return USDU_OK;
}

int usdu_png_base64_u8(const uint8_t* src_dev, int B, int H, int W, int C, uint8_t* staging_dev, char* text_dev,
                       void* stream) {
    USDU_REQUIRE(B >= 0 && B <= 65535, "usdu_png_base64_u8: batch %d outside [0, 65535]", B);
    PngGeom g;
    const int s = png_geom(H, W, C, &g);
    if (s != USDU_OK) return s;
    if (B == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && staging_dev && text_dev, "usdu_png_base64_u8: null pointer");
    USDU_REQUIRE(((uintptr_t)staging_dev & 15) == 0 && ((uintptr_t)text_dev & 3) == 0,
                 "usdu_png_base64_u8: staging must be 16-byte and text 4-byte aligned");
    USDU_REQUIRE(g.nblk < (1 << 30), "usdu_png_base64_u8: frame too large");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = kSpan + 4;
    int r = raise_smem_limit((const void*)png_idat_kernel, smem);
    if (r != USDU_OK) return r;
    png_idat_kernel<<<dim3((unsigned)g.nblk, (unsigned)B), kPngThreads, smem, st>>>(
        src_dev, (int64_t)H * g.row_bytes, (uint32_t)g.row_bytes, (uint32_t)g.rowlen, g.raw, (int)g.nblk, staging_dev,
        g.stride, g.png_area);
    USDU_CUDA(cudaGetLastError());
    png_frame_kernel<<<B, kPngThreads, 0, st>>>(H, W, C, g.raw, (int)g.nblk, staging_dev, g.stride, g.png_len,
                                                g.png_area);
    USDU_CUDA(cudaGetLastError());
    const int64_t units = (g.png_len + 11) / 12;
    const int64_t total = units * B;
    const int64_t blocks = (total + kPngThreads - 1) / kPngThreads;
    const int grid = (int)(blocks < (int64_t)grid_sms() * 16 ? blocks : (int64_t)grid_sms() * 16);
    png_base64_kernel<<<grid, kPngThreads, 0, st>>>(staging_dev, g.stride, g.png_len, units, total, text_dev,
                                                    g.text_len);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

int usdu_png_encode_u8(const uint8_t* src_dev, int B, int H, int W, int C, const uint8_t* template_dev, int64_t png_len,
                       const int64_t* runs_dev, int n_runs, const int64_t* chunks_dev, int n_chunks,
                       const int64_t* adler_at, uint8_t* scratch_dev, uint8_t* dst_dev, void* stream) {
    USDU_REQUIRE(B >= 0 && B <= 65535, "usdu_png_encode_u8: batch %d outside [0, 65535]", B);
    USDU_REQUIRE(C == 3, "usdu_png_encode_u8: %d channels: only RGB frames are encoded", C);
    USDU_REQUIRE(H >= 1 && W >= 1, "usdu_png_encode_u8: empty frame %dx%d", W, H);
    USDU_REQUIRE((int64_t)W * C <= USDU_PNG_MAX_ROW_BYTES, "usdu_png_encode_u8: rows of %lld bytes (at most %d)",
                 (long long)W * C, USDU_PNG_MAX_ROW_BYTES);
    const int64_t rowlen = (int64_t)W * C + 1, raw = (int64_t)H * rowlen;
    USDU_REQUIRE(png_len > raw && n_runs >= 1 && n_chunks >= 1,
                 "usdu_png_encode_u8: layout of %lld bytes, %d runs, %d chunks for a stream of %lld bytes",
                 (long long)png_len, n_runs, n_chunks, (long long)raw);
    USDU_REQUIRE(adler_at, "usdu_png_encode_u8: null pointer");
    AdlerAt at;
    for (int i = 0; i < 4; ++i) {
        USDU_REQUIRE(adler_at[i] >= 0 && adler_at[i] < png_len, "usdu_png_encode_u8: Adler byte %d at %lld", i,
                     (long long)adler_at[i]);
        at.p[i] = adler_at[i];
    }
    if (B == 0) return USDU_OK;
    USDU_REQUIRE(src_dev && template_dev && runs_dev && chunks_dev && scratch_dev && dst_dev,
                 "usdu_png_encode_u8: null pointer");
    USDU_REQUIRE(((uintptr_t)scratch_dev & 15) == 0, "usdu_png_encode_u8: scratch must be 16-byte aligned");
    const int64_t parts_at = (raw + 15) / 16 * 16;
    const int64_t stride = parts_at + 8 * (int64_t)H + 16;
    cudaStream_t st = (cudaStream_t)stream;
    png_filter_kernel<<<dim3((unsigned)((H + kRowsPerCta - 1) / kRowsPerCta), (unsigned)B), kPngThreads, 0, st>>>(
        src_dev, H, (uint32_t)(W * C), scratch_dev, stride, parts_at);
    USDU_CUDA(cudaGetLastError());
    png_adler_frame_kernel<<<B, kPngThreads, 0, st>>>(H, (uint32_t)rowlen, scratch_dev, stride, parts_at, template_dev,
                                                      png_len, chunks_dev, n_chunks, dst_dev);
    USDU_CUDA(cudaGetLastError());
    const size_t smem = kSpan + 4;
    int r = raise_smem_limit((const void*)png_chunk_kernel, smem);
    if (r != USDU_OK) return r;
    png_chunk_kernel<<<dim3((unsigned)n_chunks, (unsigned)B), kPngThreads, smem, st>>>(
        scratch_dev, stride, parts_at + 8 * (int64_t)H, template_dev, png_len, runs_dev, n_runs, chunks_dev, at,
        dst_dev);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

}  // extern "C"
