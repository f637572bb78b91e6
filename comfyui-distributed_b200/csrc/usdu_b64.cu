// usdu_b64.cu -- the collector master's job_complete checks on the device: the image field's base64 text decoded, and
// the O(bytes) part of http_master.parse_png over the decoded PNG (include/usdu_b200.h, usdu_b64_png_check).
//
// A worker posts each frame as base64 of a level-0 PNG inside a JSON envelope.  The route handler used to run
// b64decode(validate=True) and parse_png on the host, on ComfyUI's event loop.  Here the text (pinned host memory,
// read in place) goes through four launches on the route's stream, and the host reads back one small table:
//   Pass 1  b64_kernel        16 characters -> 12 bytes per thread; the verdict's three reductions (a byte outside
//                             the alphabet, the first '=', the last other byte) by warp reduction + one atomic per warp.
//   Pass 2  walk_kernel       one thread: Python's strict a2b_base64 verdict and the decoded length from those three
//                             words; the chunk headers from byte 8 on; the stored-block headers of the zlib stream
//                             through the IDAT chunks; the file's first bytes (IHDR and the chunks before IDAT, whose
//                             CRCs the host checks).
//   Pass 3  block_sums_kernel one CTA per stored block (grid-stride): the block's Adler-32 partials.
//   Pass 4  finish_kernel     one CTA: the Adler-32 of the stored data from the partials; the largest filter byte over
//                             the IHDR's rows, each found through the block and IDAT tables.
// The host (http_collector.check_png_tables) replays parse_png's walk over the chunk and block entries, raising its
// reasons in its order, and takes the Adler-32 and the filter verdict from the table.  Pass 2 is serial: one dependent
// load per chunk and per block header, a few hundred of each for a 4K frame.
#include "usdu_common.cuh"

namespace usdu {
namespace {

constexpr int kB64Threads = 256;
constexpr uint32_t kAdlerMod = 65521u;
constexpr int kChunkBase = USDU_B64_HEAD_WORDS;
constexpr int kBlockBase = kChunkBase + 4 * USDU_B64_MAX_CHUNKS;
constexpr int kPrefixBase = kBlockBase + 4 * USDU_B64_MAX_BLOCKS;
constexpr uint32_t kIDAT = 0x49444154u, kIEND = 0x49454E44u, kIHDR = 0x49484452u;

// value of a base64 character: 0..63, 64 for '=', 65 for anything else
__device__ __forceinline__ uint32_t b64_value(uint32_t c) {
    if (c >= 'A' && c <= 'Z') return c - 'A';
    if (c >= 'a' && c <= 'z') return c - 'a' + 26;
    if (c >= '0' && c <= '9') return c - '0' + 52;
    if (c == '+') return 62;
    if (c == '/') return 63;
    return c == '=' ? 64 : 65;
}

// head[0] |= bad, head[1] = max(n - first '='), head[2] = max(last other byte + 1); all zero on entry
__global__ void __launch_bounds__(kB64Threads) b64_kernel(const uint8_t* __restrict__ text, uint32_t n,
                                                          uint8_t* __restrict__ out, unsigned long long* head) {
    const uint32_t units = (n + 15) / 16;
    uint32_t bad = 0, eq = 0, last = 0;                   // eq: n - first '=' index seen by this thread
    const uint32_t step = gridDim.x * blockDim.x;
    for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < units; u += step) {
        uint8_t c[16];
        const uint32_t i0 = 16 * u;
        if (i0 + 16 <= n) {
            const uint4 w = *reinterpret_cast<const uint4*>(text + i0);
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int k = 0; k < 16; ++k) c[k] = (uint8_t)(ws[k >> 2] >> (8 * (k & 3)));
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) c[k] = i0 + k < n ? text[i0 + k] : (uint8_t)'=';   // past the end: no data
        }
        uint32_t v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const uint32_t x = b64_value(c[k]);
            const bool inside = i0 + k < n;
            if (inside && x == 65) bad = 1;
            if (inside && x == 64 && eq == 0) eq = n - (i0 + k);
            if (inside && x < 64) last = i0 + k + 1;
            v[k] = x < 64 ? x : 0;                        // '=' and refused bytes decode as 0 (never used)
        }
        uint32_t* o = reinterpret_cast<uint32_t*>(out + 12 * (size_t)u);
        uint8_t b[12];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint32_t t = (v[4 * q] << 18) | (v[4 * q + 1] << 12) | (v[4 * q + 2] << 6) | v[4 * q + 3];
            b[3 * q] = (uint8_t)(t >> 16); b[3 * q + 1] = (uint8_t)(t >> 8); b[3 * q + 2] = (uint8_t)t;
        }
#pragma unroll
        for (int q = 0; q < 3; ++q)
            o[q] = b[4 * q] | (b[4 * q + 1] << 8) | (b[4 * q + 2] << 16) | ((uint32_t)b[4 * q + 3] << 24);
    }
    bad = __reduce_or_sync(0xffffffffu, bad);
    eq = __reduce_max_sync(0xffffffffu, eq);
    last = __reduce_max_sync(0xffffffffu, last);
    if ((threadIdx.x & 31) == 0) {
        if (bad) atomicMax(&head[0], 1ull);
        if (eq) atomicMax(&head[1], (unsigned long long)eq);
        if (last) atomicMax(&head[2], (unsigned long long)last);
    }
}

__device__ __forceinline__ uint32_t be32(const uint8_t* p) {
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}

// the IDAT chunk holding stream byte s: the last of the n entries (stream start in word 3) starting at or before s
__device__ __forceinline__ int find_idat(const int64_t* ch, int n, int64_t s) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int m = (lo + hi + 1) >> 1;
        if (ch[4 * m + 3] <= s) lo = m; else hi = m - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(128) walk_kernel(const uint8_t* __restrict__ png, int64_t n, int64_t* tab) {
    __shared__ int64_t m_sh;
    int64_t* head = tab;
    if (threadIdx.x == 0) {
        const int64_t bad = head[0], first = n - head[1], last = head[2];
        head[1] = first;
        int64_t m = -1;
        const int64_t q = first % 4, p = n - first;
        if (!bad && last <= first && !(n > 0 && first == 0) &&
            (q == 0 || (q == 2 && p == 2) || (q == 3 && p == 1)))
            m = 3 * (first / 4) + (q == 0 ? 0 : q - 1);
        head[3] = m;
        for (int k = 4; k < USDU_B64_HEAD_WORDS; ++k) head[k] = 0;
        head[6] = head[7] = head[11] = head[12] = head[13] = -1;
        m_sh = m;
    }
    __syncthreads();
    const int64_t m = m_sh;
    uint8_t* prefix = reinterpret_cast<uint8_t*>(tab + kPrefixBase);
    const int64_t np = m < USDU_B64_PREFIX_BYTES ? m : USDU_B64_PREFIX_BYTES;
    for (int64_t i = threadIdx.x; i < np; i += blockDim.x) prefix[i] = png[i];
    if (threadIdx.x != 0 || m < 8) return;

    // chunks
    int64_t* ch = tab + kChunkBase;
    int64_t pos = 8, stream = 0;
    int nc = 0, idat0 = -1, nidat = 0, code = USDU_B64_CHUNKS_FULL;
    while (nc < USDU_B64_MAX_CHUNKS) {
        if (pos + 8 > m) { code = USDU_B64_CHUNKS_SHORT; break; }
        const int64_t len = be32(png + pos);
        const uint32_t type = be32(png + pos + 4);
        int64_t* e = ch + 4 * nc;
        e[0] = pos; e[1] = len; e[2] = type; e[3] = -1;
        ++nc;
        const int64_t body = pos + 8;
        if (len > 0x7FFFFFFF || body + len + 4 > m) { code = USDU_B64_CHUNKS_PAST_END; break; }
        if (nc == 1 && type == kIHDR && len == 13) {
            const uint8_t* h = png + body;
            const int64_t W = be32(h), H = be32(h + 4);
            const int depth = h[8], color = h[9];
            const int C = color == 0 ? 1 : color == 2 ? 3 : color == 4 ? 2 : color == 6 ? 4 : 0;
            if (depth == 8 && C && W >= 1 && H >= 1 && W * C <= USDU_PNG_MAX_ROW_BYTES) head[6] = H * (1 + W * C);
        }
        if (type == kIDAT) {
            if (idat0 < 0) idat0 = nc - 1;
            e[3] = stream;
            stream += len;
            ++nidat;
        } else if (nidat) {
            code = USDU_B64_CHUNKS_AFTER_IDAT;
            break;
        } else if (type == kIEND) {
            code = USDU_B64_CHUNKS_IEND;
            break;
        }
        pos = body + len + 4;
    }
    head[4] = nc;
    head[5] = code;
    head[8] = stream;
    head[16] = idat0;
    head[17] = nidat;
    if (code != USDU_B64_CHUNKS_AFTER_IDAT) return;

    // stored blocks, through the IDAT chunks
    const int64_t* id = ch + 4 * idat0;
    int cur = 0;
    auto at = [&](int64_t s) -> uint32_t {                 // stream byte s < stream; s only grows
        while (cur + 1 < nidat && id[4 * (cur + 1) + 3] <= s) ++cur;
        return png[id[4 * cur] + 8 + (s - id[4 * cur + 3])];
    };
    int64_t* bl = tab + kBlockBase;
    int nb = 0;
    int64_t raw = 0;
    int bcode = USDU_B64_BLOCKS_FULL;
    if (stream < 2) {
        bcode = USDU_B64_BLOCKS_SHORT;
    } else {
        const uint32_t cmf = at(0), flg = at(1);
        head[7] = cmf | (flg << 8);
        if ((cmf & 0x0F) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 != 0 || (flg & 0x20)) {
            bcode = USDU_B64_BLOCKS_ZLIB;
        } else {
            int64_t s = 2;
            while (nb < USDU_B64_MAX_BLOCKS) {
                if (s + 1 > stream) { bcode = USDU_B64_BLOCKS_SHORT; break; }
                const uint32_t hb = at(s);
                int64_t* e = bl + 4 * nb;
                e[0] = s; e[1] = hb; e[2] = raw; e[3] = 0;
                if (((hb >> 1) & 3) != 0) { ++nb; bcode = USDU_B64_BLOCKS_COMPRESSED; break; }
                if (s + 5 > stream) { bcode = USDU_B64_BLOCKS_SHORT; break; }
                const uint32_t ln = at(s + 1) | (at(s + 2) << 8), nln = at(s + 3) | (at(s + 4) << 8);
                e[1] = hb | ((int64_t)ln << 8) | ((int64_t)nln << 24);
                ++nb;
                if ((ln ^ nln) != 0xFFFF) { bcode = USDU_B64_BLOCKS_LEN; break; }
                s += 5;
                if (s + ln > stream) { bcode = USDU_B64_BLOCKS_SHORT; break; }
                raw += ln;
                s += ln;
                if (hb & 1) {
                    bcode = USDU_B64_BLOCKS_FINAL;
                    head[15] = s;
                    if (s + 4 <= stream) head[11] = (at(s) << 24) | (at(s + 1) << 16) | (at(s + 2) << 8) | at(s + 3);
                    break;
                }
            }
        }
    }
    head[9] = nb;
    head[10] = bcode;
    head[14] = raw;
}

__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    return v;
}

// block b's data: s1 = sum d, s2 = sum (LEN - j) d_j, both mod 65521, into its entry's word 3
__global__ void __launch_bounds__(kB64Threads) block_sums_kernel(const uint8_t* __restrict__ png, int64_t* tab) {
    __shared__ unsigned long long r1[kB64Threads / 32], r2[kB64Threads / 32];
    const int64_t* head = tab;
    if (head[10] != USDU_B64_BLOCKS_FINAL) return;
    const int nb = (int)head[9], nidat = (int)head[17];
    const int64_t* id = tab + kChunkBase + 4 * head[16];
    int64_t* bl = tab + kBlockBase;
    const int tid = threadIdx.x;
    for (int b = blockIdx.x; b < nb; b += gridDim.x) {
        const int64_t ln = (bl[4 * b + 1] >> 8) & 0xFFFF;
        int64_t s = bl[4 * b] + 5, done = 0;
        unsigned long long s1 = 0, s2 = 0;
        int c = find_idat(id, nidat, s);
        while (done < ln) {
            while (id[4 * c + 3] + id[4 * c + 1] <= s) ++c;           // skip chunks that end at or before s
            const int64_t take = min(ln - done, id[4 * c + 3] + id[4 * c + 1] - s);
            const uint8_t* p = png + id[4 * c] + 8 + (s - id[4 * c + 3]);
            for (int64_t j = tid; j < take; j += kB64Threads) {
                const uint32_t d = p[j];
                s1 += d;
                s2 += (unsigned long long)(ln - done - j) * d;
            }
            done += take;
            s += take;
        }
        s1 = warp_sum64(s1);
        s2 = warp_sum64(s2);
        if ((tid & 31) == 0) { r1[tid >> 5] = s1; r2[tid >> 5] = s2; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long a = 0, q = 0;
            for (int w = 0; w < kB64Threads / 32; ++w) { a += r1[w]; q += r2[w]; }
            bl[4 * b + 3] = (int64_t)((a % kAdlerMod) | ((q % kAdlerMod) << 32));
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kB64Threads) finish_kernel(const uint8_t* __restrict__ png, int64_t* tab) {
    __shared__ unsigned long long r1[kB64Threads / 32], r2[kB64Threads / 32];
    __shared__ unsigned int filt;
    int64_t* head = tab;
    if (head[10] != USDU_B64_BLOCKS_FINAL) return;
    const int nb = (int)head[9], nidat = (int)head[17];
    const int64_t raw = head[14];
    const int64_t* id = tab + kChunkBase + 4 * head[16];
    const int64_t* bl = tab + kBlockBase;
    const int tid = threadIdx.x;
    if (tid == 0) filt = 0;
    // Adler-32 of the concatenated block data: A = 1 + sum s1_b, B = |D| + sum_b [s2_b + (|D| - a_b - L_b) s1_b]
    unsigned long long A = 0, Bs = 0;
    for (int b = tid; b < nb; b += kB64Threads) {
        const unsigned long long part = (unsigned long long)bl[4 * b + 3];
        const unsigned long long s1 = part & 0xFFFFFFFFull, s2 = part >> 32;
        const int64_t L = (bl[4 * b + 1] >> 8) & 0xFFFF;
        const unsigned long long after = (unsigned long long)(raw - bl[4 * b + 2] - L) % kAdlerMod;
        A = (A + s1) % kAdlerMod;
        Bs = (Bs + s2 + after * s1) % kAdlerMod;
    }
    A = warp_sum64(A);
    Bs = warp_sum64(Bs);
    if ((tid & 31) == 0) { r1[tid >> 5] = A; r2[tid >> 5] = Bs; }
    __syncthreads();
    // filter bytes: row r's is data byte r * rowlen, in the last block starting at or before it
    const int64_t raw_len = head[6];
    const bool scan = raw_len > 0 && raw >= raw_len;
    if (scan) {
        // H and the row length from head[6] alone are ambiguous: re-read IHDR (the walk checked it) from the prefix
        const uint8_t* ih = reinterpret_cast<const uint8_t*>(tab + kPrefixBase) + 16;
        const int64_t W = be32(ih), H = be32(ih + 4);
        const int color = ih[9];
        const int64_t C = color == 0 ? 1 : color == 2 ? 3 : color == 4 ? 2 : 4;
        const int64_t rowlen = 1 + W * C;
        unsigned int mx = 0;
        for (int64_t r = tid; r < H; r += kB64Threads) {
            const int64_t q = r * rowlen;
            int lo = 0, hi = nb - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (bl[4 * mid + 2] <= q) lo = mid; else hi = mid - 1;
            }
            const int64_t s = bl[4 * lo] + 5 + (q - bl[4 * lo + 2]);
            const int c = find_idat(id, nidat, s);
            const unsigned int v = png[id[4 * c] + 8 + (s - id[4 * c + 3])];
            mx = v > mx ? v : mx;
        }
        mx = __reduce_max_sync(0xffffffffu, mx);
        if ((tid & 31) == 0) atomicMax(&filt, mx);
    }
    __syncthreads();
    if (tid != 0) return;
    for (int w = 1; w < kB64Threads / 32; ++w) { A += r1[w]; Bs += r2[w]; }
    const uint32_t s1 = (uint32_t)((1 + A) % kAdlerMod);
    const uint32_t s2 = (uint32_t)(((unsigned long long)raw % kAdlerMod + Bs) % kAdlerMod);
    head[12] = (int64_t)(((uint64_t)s2 << 16) | s1);
    head[13] = scan ? (int64_t)filt : -1;
}

}  // namespace
}  // namespace usdu

using namespace usdu;

extern "C" {

int usdu_b64_png_check(const char* text, int64_t n, uint8_t* png_dev, int64_t* table_dev, void* stream) {
    USDU_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) - 16, "usdu_b64_png_check: %lld text bytes", (long long)n);
    USDU_REQUIRE(text && png_dev && table_dev, "usdu_b64_png_check: null pointer");
    USDU_REQUIRE(((uintptr_t)text & 15) == 0 && ((uintptr_t)png_dev & 15) == 0 && ((uintptr_t)table_dev & 7) == 0,
                 "usdu_b64_png_check: text and png must be 16-byte, the table 8-byte aligned");
    // pinned host text is read through its device alias (the same address under UVA, cudaHostAlloc)
    cudaPointerAttributes pa;
    USDU_CUDA(cudaPointerGetAttributes(&pa, text));
    const uint8_t* src = reinterpret_cast<const uint8_t*>(text);
    if (pa.type == cudaMemoryTypeHost) {
        void* alias = nullptr;
        USDU_CUDA(cudaHostGetDevicePointer(&alias, const_cast<char*>(text), 0));
        src = static_cast<const uint8_t*>(alias);
    } else {
        USDU_REQUIRE(pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged,
                     "usdu_b64_png_check: text is neither device nor pinned host memory");
    }
    cudaStream_t st = (cudaStream_t)stream;
    USDU_CUDA(cudaMemsetAsync(table_dev, 0, 3 * sizeof(int64_t), st));
    const int64_t units = (n + 15) / 16;
    const int64_t need = (units + kB64Threads - 1) / kB64Threads;
    const int64_t cap = (int64_t)grid_sms() * 8;
    const int grid = (int)(need < 1 ? 1 : need < cap ? need : cap);
    b64_kernel<<<grid, kB64Threads, 0, st>>>(src, (uint32_t)n, png_dev, reinterpret_cast<unsigned long long*>(table_dev));
    USDU_CUDA(cudaGetLastError());
    walk_kernel<<<1, 128, 0, st>>>(png_dev, n, table_dev);
    USDU_CUDA(cudaGetLastError());
    const int sums = 4 * grid_sms() < USDU_B64_MAX_BLOCKS ? 4 * grid_sms() : USDU_B64_MAX_BLOCKS;
    block_sums_kernel<<<sums, kB64Threads, 0, st>>>(png_dev, table_dev);
    USDU_CUDA(cudaGetLastError());
    finish_kernel<<<1, kB64Threads, 0, st>>>(png_dev, table_dev);
    USDU_CUDA(cudaGetLastError());
    return USDU_OK;
}

}  // extern "C"
