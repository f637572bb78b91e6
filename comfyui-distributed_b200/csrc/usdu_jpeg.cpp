// usdu_jpeg.cpp -- the host half of the baseline JPEG decode: marker parse and Huffman (entropy) decode.
//
// A master's routes accept a JPEG only where PIL's Image.open(...).convert("RGB") (libjpeg-turbo, default settings)
// gives pixels this library reproduces bit for bit on the device (csrc/usdu_jpeg_decode.cu): SOF0/SOF1, 8-bit, one
// scan holding every component, 1 component or 3 with the first at h, v in {1, 2} and the others 1x1.  The parse is
// strict: every check below that fails refuses the file, also where libjpeg would only warn, so a file taken here is
// never one whose pixels depend on libjpeg's recovery from damage.
//   * SOI, then markers with in-bounds lengths: APPn / COM skipped (APP0 "JFIF" and APP14 "Adobe" read for the colour
//     space, as libjpeg's default_decompress_parms), DQT (8- or 16-bit entries, Tq < 4), DHT (Tc < 2, Th < 4, at most
//     256 codes, no code overflow, DC symbols <= 15), DRI, one SOF0/1, then SOS; any other marker refuses.
//   * SOS: Ns = Nf in frame order, defined tables, Ss = 0, Se = 63, Ah = Al = 0.
//   * the entropy-coded data: every Huffman code valid, no AC coefficient index past 63, exactly the frame's MCU count,
//     RST0..7 in sequence after every restart interval with no byte between the last MCU and the marker, then EOI,
//     then the end of the data.
//   * sides of at most 65,500 (libjpeg's JPEG_MAX_DIMENSION) and at most 2 * 89,478,485 pixels (PIL's
//     decompression-bomb limit refuses larger images);
//   * no APPn segment PIL's Python header parse raises on (check_app).
// The coefficients are written as int16 blocks in natural (row-major) order, per component a raster of blocks over the
// MCU-padded component (the layout usdu_jpeg_decode_u8 reads).  The DC value is the 32-bit running sum truncated to
// 16 bits, as libjpeg stores it.
#include <stdint.h>
#include <string.h>

#include "../../include/usdu_b200.h"

namespace usdu {
void set_error(const char* fmt, ...);
}

namespace {

constexpr int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
constexpr int kMaxSide = 65500;                    // libjpeg's JPEG_MAX_DIMENSION: JERR_IMAGE_TOO_BIG above
constexpr int64_t kMaxPixels = 2LL * 89478485;    // PIL.Image.MAX_IMAGE_PIXELS * 2: DecompressionBombError above

struct Huff {
    bool defined = false;
    int32_t maxcode[18];      // largest code of each length (-1: none), [17] sentinel
    int32_t valoff[17];       // symbol index of the first code of each length minus that code
    uint8_t vals[256];
    int16_t look[512];        // 9-bit lookahead: (length << 8) | symbol, or -1
};

struct Frame {
    int W = 0, H = 0, nc = 0, colour = 0, restart = 0;
    int id[3], h[3], v[3], tq[3], td[3], ta[3];
    int mcux = 0, mcuy = 0;
    int bw[3], bh[3];
    int64_t blocks = 0, scan = 0;                 // total blocks; offset of the first entropy-coded byte
    uint16_t q[4][64];
    bool qdef[4] = {false, false, false, false};
    Huff dc[4], ac[4];
};

#define FAIL(...)                       \
    do {                                \
        usdu::set_error(__VA_ARGS__);   \
        return USDU_ERR_INVALID;        \
    } while (0)

int build_huff(Huff& t, const uint8_t* counts, const uint8_t* syms, bool is_dc) {
    int n = 0;
    for (int l = 0; l < 16; ++l) n += counts[l];
    if (n > 256) FAIL("bad Huffman table: %d codes", n);
    for (int i = 0; i < n; ++i) {
        if (is_dc && syms[i] > 15) FAIL("bad Huffman table: DC symbol %d", syms[i]);
        t.vals[i] = syms[i];
    }
    for (int i = 0; i < 512; ++i) t.look[i] = -1;
    int32_t code = 0;
    int k = 0;
    for (int l = 1; l <= 16; ++l) {
        const int c = counts[l - 1];
        t.valoff[l] = k - code;
        for (int i = 0; i < c; ++i, ++k, ++code) {
            if (l <= 9) {
                const int span = 1 << (9 - l);
                for (int j = 0; j < span; ++j) t.look[(code << (9 - l)) | j] = (int16_t)((l << 8) | t.vals[k]);
            }
        }
        if (code >= (1 << l)) FAIL("bad Huffman table: code overflow");   // no all-ones code (libjpeg)
        t.maxcode[l] = c ? code - 1 : -1;
        code <<= 1;
    }
    t.maxcode[17] = 0x7fffffff;
    t.defined = true;
    return USDU_OK;
}

inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

inline bool starts(const uint8_t* s, int sl, const char* sig, int n) { return sl >= n && memcmp(s, sig, n) == 0; }

// PIL reads some APPn segments in Python before libjpeg sees the file (JpegImagePlugin.APP, SOF, jpeg_factory) and
// raises on these: "JFIF" APP0 and "Adobe" APP14 shorter than the 16-bit version at byte 5; an "ICC_PROFILE\0" APP2
// without its sequence and count bytes; a "Photoshop 3.0\0" APP13 whose 8BIM resource ends right after its code.  An
// "MPF\0" APP2 makes PIL read the file as an MPO, a container of several images: refused as well.
int check_app(int m, const uint8_t* s, int sl) {
    if ((m == 0xE0 && starts(s, sl, "JFIF", 4) && sl < 7) || (m == 0xEE && starts(s, sl, "Adobe", 5) && sl < 7))
        FAIL("JPEG: APP%d segment too short for its header", m - 0xE0);
    if (m == 0xE2 && starts(s, sl, "ICC_PROFILE", 12) && sl < 14) FAIL("JPEG: short ICC_PROFILE segment");
    if (m == 0xE2 && starts(s, sl, "MPF", 4)) FAIL("unsupported JPEG: MPF (multi-picture) segment");
    if (m == 0xED && starts(s, sl, "Photoshop 3.0", 14)) {
        int64_t at = 14;                         // PIL's 8BIM walk; its struct.error cases end the walk quietly
        while (at + 4 <= sl && memcmp(s + at, "8BIM", 4) == 0) {
            at += 4;
            if (at + 2 > sl) break;
            const int code = be16(s + at);
            at += 2;
            if (at >= sl) FAIL("JPEG: truncated Photoshop resource");
            at += 1 + s[at];
            at += at & 1;
            if (at + 4 > sl) break;
            const int64_t size = ((int64_t)s[at] << 24) | (s[at + 1] << 16) | (s[at + 2] << 8) | s[at + 3];
            at += 4;
            if (code == 0x03ED && at + 14 > sl) break;          // ResolutionInfo read short: struct.error
            if (code == 0x03ED && size < 14) break;
            at += size;
            at += at & 1;
        }
    }
    return USDU_OK;
}

int parse(const uint8_t* d, int64_t n, Frame& f) {
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) FAIL("not a JPEG file");
    int64_t pos = 2;
    bool sof = false, jfif = false, adobe = false;
    int transform = -1;
    for (;;) {
        if (pos >= n || d[pos] != 0xFF) FAIL("JPEG: no marker at byte %lld", (long long)pos);
        while (pos < n && d[pos] == 0xFF) ++pos;     // fill bytes
        if (pos >= n) FAIL("JPEG: truncated marker");
        const int m = d[pos++];
        if (m == 0xD8 || m == 0xD9 || m == 0x01 || (m >= 0xD0 && m <= 0xD7) || m == 0x00)
            FAIL("JPEG: marker 0x%02X before the scan", m);
        if (pos + 2 > n) FAIL("JPEG: truncated segment length");
        const int len = be16(d + pos);
        if (len < 2 || pos + len > n) FAIL("JPEG: segment 0x%02X runs past the end", m);
        const uint8_t* s = d + pos + 2;
        const int sl = len - 2;
        if (m >= 0xE0 && m <= 0xEF) {
            const int r = check_app(m, s, sl);
            if (r != USDU_OK) return r;
            if (m == 0xE0 && sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;
            if (m == 0xEE && sl >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = true, transform = s[11];
        } else if (m == 0xFE) {
        } else if (m == 0xDB) {
            int i = 0;
            while (i < sl) {
                const int pq = s[i] >> 4, tq = s[i] & 15;
                if (pq > 1 || tq > 3) FAIL("JPEG: bad DQT table %d precision %d", tq, pq);
                const int need = 1 + 64 * (pq + 1);
                if (i + need > sl) FAIL("JPEG: DQT runs past its segment");
                for (int k = 0; k < 64; ++k)
                    f.q[tq][kZigzag[k]] = (uint16_t)(pq ? be16(s + i + 1 + 2 * k) : s[i + 1 + k]);
                f.qdef[tq] = true;
                i += need;
            }
        } else if (m == 0xC4) {
            int i = 0;
            while (i < sl) {
                if (i + 17 > sl) FAIL("JPEG: DHT runs past its segment");
                const int tc = s[i] >> 4, th = s[i] & 15;
                if (tc > 1 || th > 3) FAIL("JPEG: bad DHT class %d index %d", tc, th);
                int cnt = 0;
                for (int l = 0; l < 16; ++l) cnt += s[i + 1 + l];
                if (i + 17 + cnt > sl) FAIL("JPEG: DHT runs past its segment");
                const int r = build_huff(tc ? f.ac[th] : f.dc[th], s + i + 1, s + i + 17, tc == 0);
                if (r != USDU_OK) return r;
                i += 17 + cnt;
            }
        } else if (m == 0xDD) {
            if (sl != 2) FAIL("JPEG: bad DRI length");
            f.restart = be16(s);
        } else if (m == 0xC0 || m == 0xC1) {
            if (sof) FAIL("JPEG: second SOF");
            sof = true;
            if (sl < 6) FAIL("JPEG: short SOF");
            if (s[0] != 8) FAIL("unsupported JPEG: %d-bit samples", s[0]);
            f.H = be16(s + 1), f.W = be16(s + 3), f.nc = s[5];
            if (f.H == 0 || f.W == 0) FAIL("unsupported JPEG: image size %dx%d", f.W, f.H);
            if (f.W > kMaxSide || f.H > kMaxSide) FAIL("JPEG: %dx%d: a side over %d", f.W, f.H, kMaxSide);
            if ((int64_t)f.W * f.H > kMaxPixels) FAIL("JPEG: %dx%d exceeds the decompression-bomb limit", f.W, f.H);
            if (f.nc != 1 && f.nc != 3) FAIL("unsupported JPEG: %d components", f.nc);
            if (sl != 6 + 3 * f.nc) FAIL("JPEG: bad SOF length");
            for (int c = 0; c < f.nc; ++c) {
                f.id[c] = s[6 + 3 * c], f.h[c] = s[7 + 3 * c] >> 4, f.v[c] = s[7 + 3 * c] & 15, f.tq[c] = s[8 + 3 * c];
                if (f.tq[c] > 3) FAIL("JPEG: bad quantisation table index");
                for (int e = 0; e < c; ++e)
                    if (f.id[e] == f.id[c]) FAIL("JPEG: duplicate component id");
            }
            if (f.h[0] < 1 || f.h[0] > 2 || f.v[0] < 1 || f.v[0] > 2) FAIL("unsupported JPEG: sampling %dx%d", f.h[0], f.v[0]);
            for (int c = 1; c < f.nc; ++c)
                if (f.h[c] != 1 || f.v[c] != 1) FAIL("unsupported JPEG: chroma sampling %dx%d", f.h[c], f.v[c]);
        } else if (m == 0xDA) {
            if (!sof) FAIL("JPEG: SOS before SOF");
            if (sl < 1 || sl != 4 + 2 * s[0]) FAIL("JPEG: bad SOS length");
            if (s[0] != f.nc) FAIL("unsupported JPEG: scan of %d of %d components", s[0], f.nc);
            for (int c = 0; c < f.nc; ++c) {
                if (s[1 + 2 * c] != f.id[c]) FAIL("unsupported JPEG: scan components out of frame order");
                f.td[c] = s[2 + 2 * c] >> 4, f.ta[c] = s[2 + 2 * c] & 15;
                if (f.td[c] > 3 || f.ta[c] > 3 || !f.dc[f.td[c]].defined || !f.ac[f.ta[c]].defined)
                    FAIL("JPEG: scan uses an undefined Huffman table");
                if (!f.qdef[f.tq[c]]) FAIL("JPEG: undefined quantisation table %d", f.tq[c]);
            }
            const uint8_t* e = s + 1 + 2 * f.nc;
            if (e[0] != 0 || e[1] != 63 || e[2] != 0) FAIL("unsupported JPEG: not a sequential scan");
            f.scan = pos + len;
            break;
        } else {
            FAIL("unsupported JPEG: marker 0x%02X", m);
        }
        pos += len;
    }
    if (f.nc == 1) {
        f.h[0] = f.v[0] = 1;                     // a single-component scan is not interleaved: one block per MCU
        f.colour = USDU_JPEG_GREY;
    } else if (jfif) {
        f.colour = USDU_JPEG_YCC;
    } else if (adobe) {
        if (transform != 0 && transform != 1) FAIL("JPEG: unknown Adobe transform %d", transform);
        f.colour = transform ? USDU_JPEG_YCC : USDU_JPEG_RGB;
    } else {
        f.colour = (f.id[0] == 82 && f.id[1] == 71 && f.id[2] == 66) ? USDU_JPEG_RGB : USDU_JPEG_YCC;
    }
    f.mcux = (f.W + 8 * f.h[0] - 1) / (8 * f.h[0]);
    f.mcuy = (f.H + 8 * f.v[0] - 1) / (8 * f.v[0]);
    f.blocks = 0;
    for (int c = 0; c < f.nc; ++c) {
        f.bw[c] = f.mcux * (c ? 1 : f.h[0]);
        f.bh[c] = f.mcuy * (c ? 1 : f.v[0]);
        f.blocks += (int64_t)f.bw[c] * f.bh[c];
    }
    return USDU_OK;
}

// Bits of the entropy-coded segment from `pos` up to the next marker, FF 00 read as FF.
struct Bits {
    const uint8_t* d;
    int64_t n, pos;
    uint64_t acc = 0;
    int cnt = 0;
    bool marker = false;      // the segment's marker was reached: no more bytes
    inline void fill() {
        while (cnt <= 56 && !marker) {
            if (pos >= n) {
                marker = true;
                break;
            }
            uint32_t b = d[pos];
            if (b == 0xFF) {
                if (pos + 1 < n && d[pos + 1] == 0x00) {
                    pos += 2;
                } else {
                    marker = true;
                    break;
                }
            } else {
                ++pos;
            }
            acc |= (uint64_t)b << (56 - cnt);
            cnt += 8;
        }
    }
    inline bool need(int k) {
        if (cnt < k) fill();
        return cnt >= k;
    }
    inline uint32_t peek(int k) const { return (uint32_t)(acc >> (64 - k)); }
    inline void skip(int k) { acc <<= k, cnt -= k; }
};

// jpeg_huff_decode: -> symbol, or -1 for a code that is no code of the table or runs into the marker
inline int decode_sym(Bits& b, const Huff& t) {
    b.need(16);
    if (b.cnt >= 9) {
        const int e = t.look[b.peek(9)];
        if (e >= 0) {
            b.skip(e >> 8);
            return e & 0xFF;
        }
    }
    for (int l = 1; l <= 16; ++l) {
        if (b.cnt < l) return -1;
        const int32_t code = (int32_t)b.peek(l);
        if (code <= t.maxcode[l]) {
            b.skip(l);
            return t.vals[t.valoff[l] + code];
        }
    }
    return -1;
}

// get_bits(s) and HUFF_EXTEND; false when the bits run into the marker
inline bool receive_extend(Bits& b, int s, int32_t* out) {
    if (s == 0) {
        *out = 0;
        return true;
    }
    if (!b.need(s)) return false;
    const int32_t r = (int32_t)b.peek(s);
    b.skip(s);
    *out = r < (1 << (s - 1)) ? r - (1 << s) + 1 : r;
    return true;
}

// The bit reader ends a segment: the bits left are less than a byte (the padding), and the marker follows at once.
inline bool at_marker(Bits& b) {
    b.fill();
    return b.cnt < 8 && b.marker && b.pos + 1 < b.n && b.d[b.pos] == 0xFF;
}

int decode(const uint8_t* d, int64_t n, const Frame& f, int16_t* out) {
    int64_t base[3];
    base[0] = 0;
    for (int c = 1; c < f.nc; ++c) base[c] = base[c - 1] + (int64_t)f.bw[c - 1] * f.bh[c - 1] * 64;
    // a single-component scan has one block per MCU, over ceil(W/8) x ceil(H/8) blocks
    const int64_t mcus = (int64_t)f.mcux * f.mcuy;
    const int per_row = f.mcux;
    Bits b{d, n, f.scan};
    int32_t last[3] = {0, 0, 0};
    int rst = 0;
    for (int64_t m = 0; m < mcus; ++m) {
        if (f.restart && m > 0 && m % f.restart == 0) {
            if (!at_marker(b) || b.d[b.pos + 1] != 0xD0 + rst) FAIL("JPEG: missing or out-of-order RST%d", rst);
            rst = (rst + 1) & 7;
            b = Bits{d, n, b.pos + 2};
            last[0] = last[1] = last[2] = 0;
        }
        const int mx = (int)(m % per_row), my = (int)(m / per_row);
        for (int c = 0; c < f.nc; ++c) {
            const int hc = c ? 1 : f.h[0], vc = c ? 1 : f.v[0];
            const Huff& dc = f.dc[f.td[c]];
            const Huff& ac = f.ac[f.ta[c]];
            for (int yy = 0; yy < vc; ++yy)
                for (int xx = 0; xx < hc; ++xx) {
                    int16_t* blk = out + base[c] + ((int64_t)(my * vc + yy) * f.bw[c] + (mx * hc + xx)) * 64;
                    memset(blk, 0, 64 * sizeof(int16_t));
                    int s = decode_sym(b, dc);
                    int32_t v;
                    if (s < 0 || !receive_extend(b, s, &v)) FAIL("JPEG: bad Huffman code (DC) in MCU %lld", (long long)m);
                    last[c] = (int32_t)((uint32_t)last[c] + (uint32_t)v);
                    blk[0] = (int16_t)last[c];
                    for (int k = 1; k < 64; ++k) {
                        const int rs = decode_sym(b, ac);
                        if (rs < 0) FAIL("JPEG: bad Huffman code (AC) in MCU %lld", (long long)m);
                        const int r = rs >> 4;
                        s = rs & 15;
                        if (s) {
                            k += r;
                            if (k > 63) FAIL("JPEG: coefficient index past 63 in MCU %lld", (long long)m);
                            if (!receive_extend(b, s, &v)) FAIL("JPEG: data ends inside MCU %lld", (long long)m);
                            blk[kZigzag[k]] = (int16_t)v;
                        } else {
                            if (r != 15) break;
                            k += 15;
                        }
                    }
                }
        }
    }
    if (!at_marker(b) || b.d[b.pos + 1] != 0xD9) FAIL("JPEG: no EOI right after the scan's last MCU");
    if (b.pos + 2 != n) FAIL("JPEG: %lld bytes after EOI", (long long)(n - b.pos - 2));
    return USDU_OK;
}

}  // namespace

extern "C" {

int usdu_jpeg_parse(const uint8_t* data, int64_t n, int64_t* info, int32_t* quant) {
    if (!data || !info || !quant || n < 0) FAIL("usdu_jpeg_parse: null pointer or negative size");
    Frame f;
    const int r = parse(data, n, f);
    if (r != USDU_OK) return r;
    for (int i = 0; i < USDU_JPEG_INFO_WORDS; ++i) info[i] = 0;
    info[USDU_JI_W] = f.W, info[USDU_JI_H] = f.H, info[USDU_JI_COMPONENTS] = f.nc;
    info[USDU_JI_H0] = f.h[0], info[USDU_JI_V0] = f.v[0], info[USDU_JI_COLOUR] = f.colour;
    info[USDU_JI_RESTART] = f.restart, info[USDU_JI_MCUX] = f.mcux, info[USDU_JI_MCUY] = f.mcuy;
    info[USDU_JI_BLOCKS] = f.blocks, info[USDU_JI_SCAN] = f.scan;
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 64; ++k) quant[c * 64 + k] = c < f.nc ? f.q[f.tq[c]][k] : 0;
    return USDU_OK;
}

int usdu_jpeg_decode_coefs(const uint8_t* data, int64_t n, int16_t* coefs, int64_t n_words) {
    if (!data || !coefs || n < 0) FAIL("usdu_jpeg_decode_coefs: null pointer or negative size");
    Frame f;
    const int r = parse(data, n, f);
    if (r != USDU_OK) return r;
    if (n_words != f.blocks * 64) FAIL("usdu_jpeg_decode_coefs: %lld words for %lld blocks", (long long)n_words,
                                       (long long)f.blocks);
    return decode(data, n, f, coefs);
}

}  // extern "C"
