// Plan.cpp -- the host-side planner of the tile path: tile geometry, the resample-table pool with its
// tensor-core fragments, feather-template classes, tile descriptors, dependency waves and the job records of the
// crop and blend kernels.  Plain host C++ behind the C ABI of include/usdu_b200.h, so that a host without Python
// can drive the whole tile path; the Python package calls the same code (planner.py via _native.py).
//
// Reference arithmetic restated here (file:line relative to robertvoy/ComfyUI-Distributed @ a91f9fb):
//   upscale/tile_ops.py:14-32      round_to_multiple (Python round(): ties to even), calculate_tiles
//   upscale/tile_ops.py:51-82      crop window of a tile (+ utils/usdu_utils.py:49-112 get_crop_region, expand_crop)
//   upscale/modes/single_gpu.py:40-64  progressive order: tile k sees the blends of every earlier tile it overlaps
// Every integer and float step follows the numpy planner it replaced (tests/planner_model.py), so the records are
// byte-identical to what it produced.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <map>
#include <new>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../include/usdu_b200.h"

namespace usdu {
void set_error(const char* fmt, ...);
int sm_count();
namespace mma {
int resident_ctas(int kernel, bool two_ksteps, int patch_w, int patch_h, int block_rows, bool use_device);
}
}  // namespace usdu

namespace {

constexpr int kMmaM = 16;            // outputs per M-tile (mma.sync.m16n8k32)
constexpr int kMmaK = 32;            // inputs per k-step
constexpr int kMmaMaxKsteps = 2;
constexpr int kCtasPerSm = 4;        // resident CTAs of the fast kernels per SM
constexpr int kDefaultSms = 132;     // H100 SXM: block shapes of plans made where no device can be queried

// Python's floor division and the ceil of an exact quotient, for any sign
int64_t floordiv(int64_t a, int64_t b) {
    int64_t q = a / b;
    if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
    return q;
}
int64_t ceildiv(int64_t a, int64_t b) { return -floordiv(-a, b); }
// Python round() of a double: half to even (the default rounding mode of nearbyint)
int64_t py_round(double v) { return (int64_t)nearbyint(v); }
int64_t round_to_multiple(int64_t value, int64_t multiple = 8) { return py_round((double)value / (double)multiple) * multiple; }
int64_t clip(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }
int32_t lo32(int64_t v) { return (int32_t)(uint32_t)(uint64_t)v; }

struct Tile {
    int64_t x, y, x1, y1, x2, y2, pw, ph, bx1, by1, bx2, by2;
    int tab_crop_h, tab_crop_v, tab_blend_h, tab_blend_v;   // indices into Plan::tables
    int64_t ew() const { return x2 - x1; }
    int64_t eh() const { return y2 - y1; }
};

struct Table {
    int n_in, n_out;
    int64_t off, packed, frag = -1;
    int ks = 0, taps = 0, job_taps = 0;
    std::vector<int64_t> first, span_lo, span_hi, end, cmax, k0;
};

// One axis of expand_crop (utils/usdu_utils.py:88-110): right/bottom by half the deficit, then left/top by what is
// still missing, then right/bottom again.
void grow(int64_t& lo, int64_t& hi, int64_t limit, int64_t target) {
    hi = std::min(hi + floordiv(target - (hi - lo), 2), limit);
    lo = std::max(lo - (target - (hi - lo)), (int64_t)0);
    hi = std::min(hi + (target - (hi - lo)), limit);
}

Tile make_tile(int64_t W, int64_t H, int64_t x, int64_t y, int64_t tw, int64_t th, int64_t padding, bool uniform) {
    // PIL draws the rectangle [x, y, x+tw, y+th] INCLUSIVE of its far corner; getbbox is exclusive, hence the +1
    // (upscale/tile_ops.py:51-54, utils/usdu_utils.py:52).
    Tile t{};
    t.x = x; t.y = y;
    t.bx1 = x; t.by1 = y;
    t.bx2 = std::min(x + tw + 1, W); t.by2 = std::min(y + th + 1, H);
    int64_t x1 = std::max(t.bx1 - padding, (int64_t)0), y1 = std::max(t.by1 - padding, (int64_t)0);
    int64_t x2 = std::min(t.bx2 + padding, W), y2 = std::min(t.by2 + padding, H);
    if (x2 < W) x2 -= 1;
    if (y2 < H) y2 -= 1;
    int64_t want_w, want_h;
    if (uniform) {
        t.pw = round_to_multiple(tw + padding);
        t.ph = round_to_multiple(th + padding);
        const int64_t cw = x2 - x1, ch = y2 - y1;
        const double crop_ratio = ch ? (double)cw / (double)ch : 1.0;
        const double proc_ratio = t.ph ? (double)t.pw / (double)t.ph : 1.0;
        if (crop_ratio > proc_ratio) {
            want_w = cw;
            want_h = proc_ratio != 0.0 ? py_round((double)cw / proc_ratio) : ch;
        } else {
            want_w = py_round((double)ch * proc_ratio);
            want_h = ch;
        }
    } else {
        t.pw = want_w = std::max((int64_t)8, ceildiv(x2 - x1, 8) * 8);
        t.ph = want_h = std::max((int64_t)8, ceildiv(y2 - y1, 8) * 8);
    }
    grow(x1, x2, W, want_w);
    grow(y1, y2, H, want_h);
    t.x1 = x1; t.y1 = y1; t.x2 = x2; t.y2 = y2;
    return t;
}

// Tensor-core fragments of a resample table (usdu_mma.cu): the axis as a banded matrix product, coefficients split into
// three 8-bit limbs (l2 signed).  -> {n_mtiles, ksteps, 0, 0} then per M-tile {k0, 0, 0, 0, fragments}, fragments = per
// (kstep, limb) 32 lanes x 4 registers in the A-operand layout of mma.m16n8k32 (lane = 4 g + t: a0 = A[g][4t..4t+3],
// a1 = A[g+8][4t..], a2 = A[g][16+4t..], a3 = A[g+8][16+4t..]); false when an M-tile needs more than kMmaMaxKsteps
// k-steps or a coefficient does not fit 24 bits (those plans keep the integer-pipe kernels).
bool build_mma_frags(const int32_t* tab, std::vector<int32_t>& out, std::vector<int64_t>& k0, int& ksteps) {
    const int n_out = tab[1], ksize = tab[2];
    const int32_t* bounds = tab + USDU_TAB_HEADER;
    const int32_t* kk = bounds + 2 * (int64_t)n_out;
    const int n_mt = (n_out + kMmaM - 1) / kMmaM;
    k0.assign(n_mt, 0);
    int64_t ks = 1;
    for (int mt = 0; mt < n_mt; ++mt) {
        const int o_lo = mt * kMmaM, o_hi = std::min(o_lo + kMmaM, n_out);
        k0[mt] = bounds[2 * o_lo] & ~3;
        int64_t end = INT64_MIN;
        for (int o = o_lo; o < o_hi; ++o) end = std::max(end, (int64_t)bounds[2 * o] + bounds[2 * o + 1]);
        ks = std::max(ks, floordiv(end - k0[mt] + kMmaK - 1, kMmaK));
    }
    if (ks > kMmaMaxKsteps) return false;
    const int K = kMmaK * (int)ks;
    std::vector<int64_t> A((size_t)n_mt * kMmaM * K, 0);   // row = output (padded), col = input - k0[mt]
    for (int o = 0; o < n_out; ++o) {
        const int64_t first = bounds[2 * o], cnt = bounds[2 * o + 1];
        for (int t = 0; t < ksize && t < cnt; ++t) A[(size_t)o * K + (first + t - k0[o / kMmaM])] = kk[(int64_t)o * ksize + t];
    }
    for (int64_t a : A)
        if ((a < 0 ? -a : a) >= (1 << 23)) return false;
    ksteps = (int)ks;
    const size_t words_per_mt = 4 + (size_t)ks * 3 * 32 * 4;
    out.assign(4 + (size_t)n_mt * words_per_mt, 0);
    out[0] = n_mt; out[1] = (int32_t)ks;
    static const int dm[4] = {0, 8, 0, 8}, dk[4] = {0, 0, 16, 16};
    for (int mt = 0; mt < n_mt; ++mt) {
        int32_t* w = out.data() + 4 + mt * words_per_mt;
        w[0] = (int32_t)k0[mt];
        w += 4;
        for (int s = 0; s < ks; ++s)
            for (int limb = 0; limb < 3; ++limb)
                for (int lane = 0; lane < 32; ++lane)
                    for (int r = 0; r < 4; ++r) {
                        const int g = lane / 4, tq = lane % 4;
                        const int64_t row = (int64_t)mt * kMmaM + g + dm[r];
                        uint32_t word = 0;
                        for (int b = 0; b < 4; ++b) {
                            const int64_t col = (int64_t)s * kMmaK + 4 * tq + dk[r] + b;
                            const uint32_t byte = (uint32_t)((A[(size_t)row * K + col] >> (8 * limb)) & 255);
                            word |= byte << (8 * b);
                        }
                        *w++ = (int32_t)word;
                    }
    }
    return true;
}

struct Plan {
    int W, H, tile_width, tile_height, padding, mask_blur;
    bool uniform;
    int64_t tw = 0, th = 0;
    std::vector<Tile> tiles;
    std::vector<int32_t> tabs;
    std::vector<Table> tables;
    std::map<std::pair<int, int>, int> tab_index;
    std::vector<int32_t> specs;            // n_classes x USDU_MASK_WORDS
    int64_t mask_pool_bytes = 0;
    std::vector<int> mask_class;
    std::vector<int32_t> desc;             // n_tiles x USDU_TILE_WORDS
    std::vector<std::vector<int>> neighbors;
    bool fast = true, mma = true;
    int gbw = 0, gbh = 0;                  // block of the generic kernels (0 = not computed yet)
    int64_t ramp = 0;

    int table(int n_in, int n_out, int* index);
    int64_t span_max(const Table& tb, int64_t block, bool aligned) const;
    void generic_block(int& bw, int& bh);
    void support(const Tile& t, int64_t s[4]) const;
    void opaque_core(const Tile& t, int64_t f[4]) const;
};

struct WorkList {
    std::vector<int32_t> items;
    int item_words = 0;
    std::vector<int32_t> cover;
    std::vector<int64_t> slots;
    int64_t total = 0, patch_w = 1, patch_h = 1, algo_bytes = 0, n_launch = -1, block_rows = 0, block_cols = 0;
    int64_t row0 = -1, row1 = -1;
    int path = 0;
    bool ks2 = false;
    int64_t n_items() const { return item_words ? (int64_t)items.size() / item_words : 0; }
};

int Plan::table(int n_in, int n_out, int* index) {
    auto it = tab_index.find({n_in, n_out});
    if (it != tab_index.end()) {
        *index = it->second;
        return USDU_OK;
    }
    // an axis that keeps its size gets a one-tap identity table (Pillow skips the pass)
    std::vector<int32_t> tab;
    if (n_in == n_out) {
        if (n_in <= 0) {
            usdu::set_error("usdu_plan_create: empty crop window axis (%d)", n_in);
            return USDU_ERR_INVALID;
        }
        tab.assign(((USDU_TAB_HEADER + 3 * (int64_t)n_in + 3) & ~(int64_t)3) + (int64_t)n_in * USDU_PACKED_ROW, 0);
        const int s = usdu_build_identity_table(n_in, tab.data());
        if (s != USDU_OK) return s;
    } else {
        const int64_t words = usdu_resample_table_words(n_in, n_out);
        if (words < 0) return (int)words;
        tab.assign(words, 0);
        const int s = usdu_build_resample_table(n_in, n_out, tab.data());
        if (s != USDU_OK) return s;
        if (tab[4]) tab.resize((size_t)tab[4] + (size_t)n_out * tab[6]);   // trim the packed section to its row stride
    }
    Table tb;
    tb.n_in = n_in; tb.n_out = n_out;
    if (tab[4] == 0) fast = false;
    tb.off = (int64_t)tabs.size();
    tabs.insert(tabs.end(), tab.begin(), tab.end());
    tb.packed = tb.off + tab[4];                                   // pool index of packed row 0 (fast kernels)
    tb.taps = tab[4] ? tab[6] - 1 : tab[3];                        // 7 or 15 staged taps per output on the fast path
    // what the job records carry: the real maximum when it is below the 7-slot row (an up-scaling LANCZOS axis uses
    // exactly 6), so the kernels can skip the always-zero last slot
    tb.job_taps = tb.taps <= USDU_FAST_TAPS ? std::min(tb.taps, std::max(tab[3], 1)) : tb.taps;
    const int32_t* b = tab.data() + USDU_TAB_HEADER;
    if (mma) {
        std::vector<int32_t> frags;
        if (!build_mma_frags(tab.data(), frags, tb.k0, tb.ks)) {
            mma = false;
        } else {
            tb.frag = (int64_t)tabs.size();                       // tables end on a multiple of 4 int32
            tabs.insert(tabs.end(), frags.begin(), frags.end());
            tabs.resize((tabs.size() + 3) & ~(size_t)3, 0);
            tb.end.resize(n_out);
            tb.cmax.resize(n_out);
            for (int o = 0; o < n_out; ++o) {
                tb.end[o] = (int64_t)b[2 * o] + b[2 * o + 1];
                tb.cmax[o] = o ? std::max(tb.cmax[o - 1], tb.end[o]) : tb.end[o];
            }
        }
    }
    tb.first.resize(n_out);
    tb.span_lo.resize(n_out);
    tb.span_hi.resize(n_out);
    for (int o = 0; o < n_out; ++o) {
        tb.first[o] = tb.span_lo[o] = b[2 * o];
        tb.span_hi[o] = (int64_t)b[2 * o] + std::max(b[2 * o + 1], tb.taps);   // [lo, hi) of the inputs per output
    }
    *index = (int)tables.size();
    tab_index[{n_in, n_out}] = *index;
    tables.push_back(std::move(tb));
    return USDU_OK;
}

// Largest input extent read by `block` consecutive outputs of an axis.
int64_t Plan::span_max(const Table& tb, int64_t block, bool aligned) const {
    const int64_t n = tb.n_out;
    int64_t best = INT64_MIN;
    for (int64_t s = 0; s < n; s += aligned ? block : 1) {
        const int64_t e = std::min(s + block, n) - 1;
        best = std::max(best, tb.span_hi[e] - tb.span_lo[s]);
    }
    return best;
}

// Block of the generic kernels: 64 x 32 unless an extreme scale (a canvas much smaller than a tile) makes the input
// patch of such a block exceed shared memory; then halve.
void Plan::generic_block(int& bw_out, int& bh_out) {
    if (!gbw) {
        int64_t bw = USDU_BLOCK_W, bh = USDU_BLOCK_H;
        while (true) {
            int64_t pw_ = INT64_MIN, ph_ = INT64_MIN;
            for (const Table& tb : tables) {
                pw_ = std::max(pw_, span_max(tb, bw, false));
                ph_ = std::max(ph_, span_max(tb, bh, false));
            }
            if (tables.empty()) pw_ = bw, ph_ = bh;
            const int64_t smem = (int64_t)USDU_BLOCK_H * USDU_BLOCK_W * 3 + ph_ * USDU_BLOCK_W * 3 + ph_ * floordiv(pw_ * 3 + 15, 16) * 16;
            if (smem <= 200 * 1024 || (bw <= 4 && bh <= 4)) break;
            if ((pw_ * bh >= ph_ * bw && bw > 4) || bh <= 4)
                bw /= 2;
            else
                bh /= 2;
        }
        gbw = (int)bw;
        gbh = (int)bh;
    }
    bw_out = gbw;
    bh_out = gbh;
}

// Window-relative bbox outside which the feather alpha is exactly 0.
void Plan::support(const Tile& t, int64_t s[4]) const {
    s[0] = std::max(t.bx1 - ramp, t.x1) - t.x1;
    s[1] = std::max(t.by1 - ramp, t.y1) - t.y1;
    s[2] = std::min(t.bx2 + ramp, t.x2) - t.x1;
    s[3] = std::min(t.by2 + ramp, t.y2) - t.y1;
}

// Window-relative box inside which the feather alpha is exactly 255: the rectangle shrunk by the ramp, except on sides
// where the rectangle touches the canvas border (edge replication keeps the mask at 255 there).
void Plan::opaque_core(const Tile& t, int64_t f[4]) const {
    int64_t fx0 = t.bx1 == 0 ? t.bx1 : t.bx1 + ramp;
    int64_t fy0 = t.by1 == 0 ? t.by1 : t.by1 + ramp;
    int64_t fx1 = t.bx2 == W ? t.bx2 : t.bx2 - ramp;
    int64_t fy1 = t.by2 == H ? t.by2 : t.by2 - ramp;
    fx0 = std::max(fx0, t.x1); fy0 = std::max(fy0, t.y1);
    fx1 = std::min(fx1, t.x2); fy1 = std::min(fy1, t.y2);
    if (fx1 <= fx0 || fy1 <= fy0) {
        f[0] = f[1] = f[2] = f[3] = 0;
        return;
    }
    f[0] = fx0 - t.x1; f[1] = fy0 - t.y1; f[2] = fx1 - t.x1; f[3] = fy1 - t.y1;
}

int build_plan(Plan* p) {
    p->tw = round_to_multiple(p->tile_width);
    p->th = round_to_multiple(p->tile_height);
    if (p->tw <= 0 || p->th <= 0) {
        usdu::set_error("tile size rounds to zero: %dx%d", p->tile_width, p->tile_height);
        return USDU_ERR_INVALID;
    }
    if (p->W <= 0 || p->H <= 0) {
        usdu::set_error("canvas must be at least 1x1, got %dx%d", p->W, p->H);
        return USDU_ERR_INVALID;
    }
    const int64_t cols = ceildiv(p->W, p->tw), rows = ceildiv(p->H, p->th);
    for (int64_t r = 0; r < rows; ++r)
        for (int64_t c = 0; c < cols; ++c)
            p->tiles.push_back(make_tile(p->W, p->H, c * p->tw, r * p->th, p->tw, p->th, p->padding, p->uniform));
    for (Tile& t : p->tiles) {
        int s;
        if ((s = p->table((int)t.ew(), (int)t.pw, &t.tab_crop_h)) != USDU_OK) return s;
        if ((s = p->table((int)t.eh(), (int)t.ph, &t.tab_crop_v)) != USDU_OK) return s;
        if ((s = p->table((int)t.pw, (int)t.ew(), &t.tab_blend_h)) != USDU_OK) return s;
        if ((s = p->table((int)t.ph, (int)t.eh(), &t.tab_blend_v)) != USDU_OK) return s;
    }
    for (const Tile& t : p->tiles)
        if (t.x1 % 4) p->mma = false;      // the tensor-core kernels stage 4-pixel chunks at 4-pixel canvas columns
    if (!p->fast) p->mma = false;

    // feather-template classes: tiles whose mask is the same window-relative image share one template
    if (p->mask_blur > 0) {
        int32_t rad;
        uint32_t ww, fw;
        const int s = usdu_box_blur_params((float)p->mask_blur, &rad, &ww, &fw);
        if (s != USDU_OK) return s;
        p->ramp = 3 * ((int64_t)rad + 1);     // 3 box passes of half-width rad+1 each
    }
    const int64_t ext = p->ramp;
    std::map<std::array<int64_t, 10>, int> classes;
    std::vector<int64_t> cls_off, cls_pitch;
    int64_t off = 0;
    for (const Tile& t : p->tiles) {
        const std::array<int64_t, 10> key = {t.bx1 - t.x1, t.bx2 - t.x1, t.ew(), std::min(t.x1, ext), std::min((int64_t)p->W - t.x2, ext),
                                             t.by1 - t.y1, t.by2 - t.y1, t.eh(), std::min(t.y1, ext), std::min((int64_t)p->H - t.y2, ext)};
        auto it = classes.find(key);
        if (it == classes.end()) {
            const int c = (int)cls_off.size();
            it = classes.emplace(key, c).first;
            const int64_t pitch = (t.ew() + 15) / 16 * 16;
            const int64_t spec[USDU_MASK_WORDS] = {p->W, p->H, t.bx1, t.by1, t.bx2, t.by2, t.x1, t.y1, t.x2, t.y2,
                                                   p->mask_blur, off, pitch, 0, 0, 0};
            for (int64_t v : spec) p->specs.push_back(lo32(v));
            cls_off.push_back(off);
            cls_pitch.push_back(pitch);
            off += pitch * t.eh();
            off = (off + 255) / 256 * 256;
        }
        p->mask_class.push_back(it->second);
    }
    p->mask_pool_bytes = std::max(off, (int64_t)256);
    if (p->mask_pool_bytes >= ((int64_t)1 << 31)) {
        usdu::set_error("feather templates exceed 2 GiB");
        return USDU_ERR_INVALID;
    }

    // tile descriptors
    p->desc.assign(p->tiles.size() * USDU_TILE_WORDS, 0);
    for (size_t i = 0; i < p->tiles.size(); ++i) {
        const Tile& t = p->tiles[i];
        int32_t* r = p->desc.data() + i * USDU_TILE_WORDS;
        r[USDU_T_X1] = (int32_t)t.x1; r[USDU_T_Y1] = (int32_t)t.y1; r[USDU_T_EW] = (int32_t)t.ew(); r[USDU_T_EH] = (int32_t)t.eh();
        r[USDU_T_PW] = (int32_t)t.pw; r[USDU_T_PH] = (int32_t)t.ph;
        r[USDU_T_MASK_OFF] = (int32_t)cls_off[p->mask_class[i]];
        r[USDU_T_MASK_PITCH] = (int32_t)cls_pitch[p->mask_class[i]];
        r[USDU_T_TAB_CROP_H] = (int32_t)p->tables[t.tab_crop_h].off;
        r[USDU_T_TAB_CROP_V] = (int32_t)p->tables[t.tab_crop_v].off;
        r[USDU_T_TAB_BLEND_H] = (int32_t)p->tables[t.tab_blend_h].off;
        r[USDU_T_TAB_BLEND_V] = (int32_t)p->tables[t.tab_blend_v].off;
        int64_t s[4], f[4];
        p->support(t, s);
        p->opaque_core(t, f);
        for (int k = 0; k < 4; ++k) {
            r[USDU_T_SUP_X0 + k] = (int32_t)s[k];
            r[USDU_T_FULL_X0 + k] = (int32_t)f[k];
        }
    }

    // tiles whose crop windows intersect (grid-bucketed, O(T * neighbours)); lists in discovery order
    const size_t T = p->tiles.size();
    p->neighbors.assign(T, {});
    if (T > 1) {
        int64_t cell = 0;
        for (const Tile& t : p->tiles) cell = std::max(cell, std::max(t.ew(), t.eh()));
        std::map<std::pair<int64_t, int64_t>, size_t> bucket_of;
        std::vector<std::vector<int>> buckets;
        for (size_t i = 0; i < T; ++i) {
            const Tile& t = p->tiles[i];
            for (int64_t gx = floordiv(t.x1, cell); gx <= floordiv(t.x2 - 1, cell); ++gx)
                for (int64_t gy = floordiv(t.y1, cell); gy <= floordiv(t.y2 - 1, cell); ++gy) {
                    auto it = bucket_of.find({gx, gy});
                    if (it == bucket_of.end()) {
                        it = bucket_of.emplace(std::make_pair(gx, gy), buckets.size()).first;
                        buckets.emplace_back();
                    }
                    buckets[it->second].push_back((int)i);
                }
        }
        std::unordered_set<uint64_t> seen;
        for (const auto& ids : buckets)
            for (size_t a = 0; a < ids.size(); ++a)
                for (size_t b = a + 1; b < ids.size(); ++b) {
                    const int i = ids[a], j = ids[b];
                    if (!seen.insert((uint64_t)(uint32_t)i << 32 | (uint32_t)j).second) continue;
                    const Tile &A = p->tiles[i], &B = p->tiles[j];
                    if (A.x1 < B.x2 && B.x1 < A.x2 && A.y1 < B.y2 && B.y1 < A.y2) {
                        p->neighbors[i].push_back(j);
                        p->neighbors[j].push_back(i);
                    }
                }
    }
    return USDU_OK;
}

// ---- kernel work lists -----------------------------------------------------------------------------------------
struct LaunchModel {
    int sm_count;        // 0 = query the device, else 132
    int mma_block_rows;  // 0 = the model's choice
};

int resident_slots(const LaunchModel& m) {
    int sms = m.sm_count;
    if (sms <= 0) {
        sms = usdu::sm_count();
        if (sms <= 0) sms = kDefaultSms;
    }
    return sms * kCtasPerSm;
}

int kernel_path(const Plan* p, int path) {
    if (path >= 2 && !p->mma) path = 1;
    if (path >= 1 && !p->fast) path = 0;
    return path;
}

// Block edge of a launch.  `extents` = (width, height) in pixels each tile covers in the launch's block space.  The block
// height is chosen by a simple wave model: cost(bh) = ceil(#CTAs / resident slots) * (bh + halo/fixed rows) -- short
// blocks give small (latency bound) launches more CTAs, and large launches avoid a nearly empty last wave.
void block_shape(Plan* p, bool use_fast, const std::vector<std::pair<int64_t, int64_t>>& extents, int64_t frames,
                 bool mma, const LaunchModel& m, int& bw_out, int& bh_out) {
    if (!use_fast) {
        p->generic_block(bw_out, bh_out);
        return;
    }
    const int64_t bw = USDU_FAST_BLOCK_W;
    bw_out = (int)bw;
    if (extents.empty()) {
        bh_out = USDU_FAST_BLOCK_H;
        return;
    }
    const int64_t slots = resident_slots(m);
    static const int mma_bh[2] = {16, 32}, fast_bh[7] = {8, 12, 16, 20, 24, 28, 32};   // M-tiles are 16 output rows
    const int forced[1] = {m.mma_block_rows};
    const int* cand = mma ? (m.mma_block_rows ? forced : mma_bh) : fast_bh;
    const int n_cand = mma ? (m.mma_block_rows ? 1 : 2) : 7;
    bool have = false;
    int64_t best_cost = 0;
    int best_bh = 0;
    for (int c = 0; c < n_cand; ++c) {
        const int64_t bh = cand[c];
        int64_t n = 0;
        for (const auto& e : extents) n += (floordiv(e.first + bw - 1, bw) + 1) * (floordiv(e.second + bh - 1, bh) + 1);   // +1: unaligned windows
        n *= frames;
        const int64_t cost = (int64_t)ceil((double)n / (double)std::max(slots, (int64_t)1)) * (bh + 12);
        if (!have || cost < best_cost || (cost == best_cost && bh > best_bh)) {
            have = true;
            best_cost = cost;
            best_bh = (int)bh;
        }
    }
    bh_out = best_bh;
}

// One axis of the tensor-core job records.  base = output index of block column / row 0 (any alignment, may be negative),
// extent = block size along the axis.  -> frag pool index, k-steps, staged start s0 (input index, multiple of 4), staged
// count, K-window need = inputs from s0 the last M-tile's window reaches.
struct MmaAxis {
    int64_t frag, ks, s0, count, need;
};
MmaAxis mma_axis(const Table& tb, int64_t base, int64_t extent) {
    const int64_t n_out = tb.n_out, n_in = tb.n_in;
    const int64_t lo = clip(base, 0, n_out - 1);
    const int64_t hi = clip(base + extent, 1, n_out);                // exclusive
    const int64_t m0 = floordiv(lo, kMmaM), m1 = floordiv(hi - 1, kMmaM);
    MmaAxis a;
    a.frag = tb.frag;
    a.ks = tb.ks;
    a.s0 = tb.k0[m0];
    const int64_t last = std::min(kMmaM * (m1 + 1), n_out) - 1;
    const int64_t stop = std::min(tb.cmax[last], n_in);
    a.count = std::max(stop - a.s0, (int64_t)1);
    a.need = tb.k0[m1] + kMmaK * tb.ks - a.s0;
    return a;
}

int64_t first_of(const Table& tb, int64_t idx) { return tb.first[clip(idx, 0, (int64_t)tb.first.size() - 1)]; }

// patch_h word of a tensor-core launch: plane rows in bits 0..15 -- the staged rows up to a multiple of 8 --, rows of the
// intermediate the kernel ALLOCATES in bits 16..31 (the K window of the last vertical M-tile may reach past the written
// rows with zero coefficients; those reads land in the byte planes behind the intermediate whenever they fit there).
int64_t mma_patch_h(int64_t max_rows, int64_t max_need_h, int64_t patch_w) {
    const int64_t plane_rows = (max_rows + 7) / 8 * 8;
    const int64_t need = (std::max(plane_rows, max_need_h) + 3) / 4 * 4;
    const int64_t overrun_bytes = (need - plane_rows) / 4 * 440 * 4;
    const int64_t planes_bytes = 3 * plane_rows * ((patch_w + 31) / 32 * 32 + 16);
    const int64_t mid_rows = overrun_bytes <= planes_bytes ? plane_rows : need;
    return plane_rows | (mid_rows << 16);
}

void set_frame(int64_t* J, int64_t pw, int64_t ph) {
    const int64_t frame = ph * pw * 3;
    J[USDU_J_PITCH] = pw * 3;
    J[USDU_J_FRAME_LO] = frame & 0xFFFFFFFF;
    J[USDU_J_FRAME_HI] = frame >> 32;
}

void store_rows(std::vector<int32_t>& dst, const std::vector<int64_t>& src) {
    dst.resize(src.size());
    for (size_t i = 0; i < src.size(); ++i) dst[i] = lo32(src[i]);
}

bool any_ks2(const std::vector<int32_t>& jobs) {
    for (size_t j = 0; j + USDU_JOB_WORDS <= jobs.size(); j += USDU_JOB_WORDS)
        if (jobs[j + USDU_J_TAPS_H] > 1 || jobs[j + USDU_J_TAPS_V] > 1) return true;
    return false;
}

int check_ids(const Plan* p, const int32_t* ids, int n, const char* what) {
    if (n < 0 || (n > 0 && !ids)) {
        usdu::set_error("%s: bad tile list (n = %d)", what, n);
        return USDU_ERR_INVALID;
    }
    for (int i = 0; i < n; ++i)
        if (ids[i] < 0 || (size_t)ids[i] >= p->tiles.size()) {
            usdu::set_error("%s: tile id %d out of range (%zu tiles)", what, ids[i], p->tiles.size());
            return USDU_ERR_INVALID;
        }
    return USDU_OK;
}

int crop_worklist(Plan* p, const int32_t* ids, int n, int B, int req_path, const LaunchModel& m, WorkList* wl) {
    const int path = kernel_path(p, req_path);
    const bool use_fast = path >= 1;
    wl->slots.resize(n);
    int64_t cur = 0;
    for (int i = 0; i < n; ++i) {
        const Tile& t = p->tiles[ids[i]];
        wl->slots[i] = cur;
        cur += (int64_t)B * t.ph * t.pw * 3;
    }
    wl->total = cur;
    std::vector<std::pair<int64_t, int64_t>> ext;
    for (int i = 0; i < n; ++i) ext.emplace_back(p->tiles[ids[i]].pw - USDU_FAST_BLOCK_W, p->tiles[ids[i]].ph);
    int bw, bh_max;
    block_shape(p, use_fast, ext, B, path == 2, m, bw, bh_max);
    std::vector<int64_t> items;     // generic items [tile, ox0, oy0, off_lo, off_hi, bh]
    int64_t pw_max = 1, ph_max = 1, nbytes = 0;
    for (int i = 0; i < n; ++i) {
        const Tile& t = p->tiles[ids[i]];
        const Table& th_ = p->tables[t.tab_crop_h];
        const Table& tv = p->tables[t.tab_crop_v];
        int64_t bh;
        if (path == 2) {
            // output rows per tensor-core crop block: 32 unless the staged input rows would not fit the 48-row TMA box
            bh = 16;
            const int64_t cands[2] = {32, 16};
            for (int c = bh_max >= 32 ? 0 : 1; c < 2; ++c) {
                int64_t worst = 0;
                for (int64_t oy0 = 0; oy0 < t.ph; oy0 += cands[c]) {
                    const int64_t mv0 = oy0 / kMmaM, mv1 = (std::min(oy0 + cands[c], t.ph) - 1) / kMmaM;
                    int64_t e = INT64_MIN;
                    for (int64_t o = kMmaM * mv0; o < std::min(kMmaM * (mv1 + 1), t.ph); ++o) e = std::max(e, tv.end[o]);
                    worst = std::max(worst, e - tv.k0[mv0]);
                }
                if (worst <= 48) {
                    bh = cands[c];
                    break;
                }
            }
        } else if (!use_fast) {
            bh = bh_max;
        } else {
            // fast path: keep the staged input rows <= 40
            bh = 8;
            for (int64_t b = bh_max; b > 7; --b)
                if (p->span_max(tv, b, true) <= 40) {
                    bh = b;
                    break;
                }
        }
        for (int64_t oy = 0; oy < t.ph; oy += bh)
            for (int64_t ox = 0; ox < t.pw; ox += bw) {
                const int64_t it[USDU_CROP_ITEM_WORDS] = {ids[i], ox, oy, wl->slots[i] & 0xFFFFFFFF, wl->slots[i] >> 32, bh};
                items.insert(items.end(), it, it + USDU_CROP_ITEM_WORDS);
            }
        pw_max = std::max(pw_max, p->span_max(th_, bw, true));
        ph_max = std::max(ph_max, p->span_max(tv, bh, true));
        nbytes += t.ew() * t.eh() * 3 + t.pw * t.ph * 3 * 4;     // u8 window read + fp32 tile write
    }
    const size_t n_items = items.size() / USDU_CROP_ITEM_WORDS;
    if (use_fast && n_items) {
        std::vector<int64_t> J(n_items * USDU_JOB_WORDS, 0);
        int64_t cols_max = INT64_MIN, need_w_max = INT64_MIN, rows_max = INT64_MIN, need_h_max = INT64_MIN;
        for (size_t j = 0; j < n_items; ++j) {
            const int64_t* it = &items[j * USDU_CROP_ITEM_WORDS];
            const Tile& t = p->tiles[it[0]];
            const Table& th_ = p->tables[t.tab_crop_h];
            const Table& tv = p->tables[t.tab_crop_v];
            const int64_t ox0 = it[1], oy0 = it[2], bh = it[5];
            int64_t* r = &J[j * USDU_JOB_WORDS];
            if (path == 2) {        // tensor-core job records (USDU_FLAG_MMA)
                const MmaAxis ah = mma_axis(th_, ox0, USDU_FAST_BLOCK_W), av = mma_axis(tv, oy0, bh);
                const int64_t cols = (ah.count + 3) & ~(int64_t)3;
                r[USDU_J_ROWS_H] = ah.frag; r[USDU_J_TAPS_H] = ah.ks;
                r[USDU_J_ROWS_V] = av.frag; r[USDU_J_TAPS_V] = av.ks;
                r[USDU_J_SRC_A] = t.x1 + ah.s0; r[USDU_J_SRC_B] = t.y1 + av.s0; r[USDU_J_LEAD] = 0;
                r[USDU_J_COLS] = cols; r[USDU_J_ROWS] = av.count; r[USDU_J_IX0] = ah.s0; r[USDU_J_IY0] = av.s0;
                r[USDU_J_CY1] = bh;                                      // block height (rows per CTA)
                cols_max = std::max(cols_max, cols); need_w_max = std::max(need_w_max, ah.need);
                rows_max = std::max(rows_max, av.count); need_h_max = std::max(need_h_max, av.need);
            } else {                // integer-pipe job records (USDU_FLAG_FAST)
                const int64_t ix0 = first_of(th_, ox0);
                const int64_t ix1 = std::min(first_of(th_, ox0 + USDU_FAST_BLOCK_W - 1) + th_.taps, (int64_t)th_.n_in);
                const int64_t iy0 = first_of(tv, oy0);
                const int64_t iy1 = std::min(first_of(tv, oy0 + bh - 1) + tv.taps, (int64_t)tv.n_in);
                const int64_t px_abs = t.x1 + ix0, lead = px_abs & 3;
                r[USDU_J_TAPS_H] = th_.job_taps; r[USDU_J_TAPS_V] = tv.job_taps;
                r[USDU_J_SRC_A] = px_abs - lead; r[USDU_J_SRC_B] = t.y1 + iy0; r[USDU_J_LEAD] = lead;
                r[USDU_J_COLS] = ix1 - ix0; r[USDU_J_ROWS] = iy1 - iy0; r[USDU_J_IX0] = ix0; r[USDU_J_IY0] = iy0;
                r[USDU_J_ROWS_H] = th_.packed; r[USDU_J_ROWS_V] = tv.packed;
            }
            r[USDU_J_OX_BASE] = ox0; r[USDU_J_N_OUT_H] = t.pw;
            r[USDU_J_OY_BASE] = oy0; r[USDU_J_N_OUT_V] = t.ph;
            r[USDU_J_DST_X] = ox0; r[USDU_J_DST_Y] = oy0;
            r[USDU_J_OFF_LO] = it[3]; r[USDU_J_OFF_HI] = it[4];
            r[USDU_J_ROWS_OUT] = std::min(bh, t.ph - oy0);
            r[USDU_J_COLS_OUT] = std::min((int64_t)USDU_FAST_BLOCK_W, t.pw - ox0);
            set_frame(r, t.pw, t.ph);
            r[USDU_J_NEXT] = -1;
        }
        if (path == 2) {
            pw_max = std::max(cols_max, need_w_max);
            ph_max = mma_patch_h(rows_max, need_h_max, pw_max);
        }
        store_rows(wl->items, J);
        wl->item_words = USDU_JOB_WORDS;
    } else {
        store_rows(wl->items, items);
        wl->item_words = USDU_CROP_ITEM_WORDS;
    }
    wl->ks2 = path == 2 && wl->item_words == USDU_JOB_WORDS && any_ks2(wl->items);
    wl->patch_w = pw_max;
    wl->patch_h = ph_max;
    wl->algo_bytes = nbytes;
    wl->block_rows = use_fast ? 0 : bh_max;
    wl->block_cols = use_fast ? 0 : bw;
    wl->path = path;
    return USDU_OK;
}

struct Pair {
    int64_t key, seq, tid;
};

int blend_worklist(Plan* p, const int32_t* ids, const int64_t* offs, int n, int src_bytes, int B, int req_path,
                   int part_i, int part_n, const LaunchModel& m, WorkList* wl) {
    const int path = kernel_path(p, req_path);
    const bool use_fast = path >= 1;
    std::vector<std::pair<int64_t, int64_t>> ext;
    for (int i = 0; i < n; ++i) {
        int64_t s[4];
        p->support(p->tiles[ids[i]], s);
        ext.emplace_back(s[2] - s[0], s[3] - s[1]);
    }
    int bw_, bh_;
    block_shape(p, use_fast, ext, B, path == 2, m, bw_, bh_);
    const int64_t bw = bw_, bh = bh_, W = p->W, H = p->H;
    const int64_t nbx = (W + bw - 1) / bw, nby = (H + bh - 1) / bh;
    int64_t lo_b = 0, hi_b = 0;
    if (part_n > 0) {
        lo_b = (nby * part_i) / part_n;
        hi_b = (nby * (part_i + 1)) / part_n;
        wl->row0 = std::min(lo_b * bh, H);
        wl->row1 = std::min(hi_b * bh, H);
    }
    std::vector<Pair> pairs;
    int64_t pw_max = 1, ph_max = 1, nbytes = 0;
    for (int s = 0; s < n; ++s) {
        const Tile& t = p->tiles[ids[s]];
        int64_t sp[4];
        p->support(t, sp);
        if (sp[2] <= sp[0] || sp[3] <= sp[1]) continue;
        const int64_t X0 = t.x1 + sp[0], Y0 = t.y1 + sp[1], X1 = t.x1 + sp[2], Y1 = t.y1 + sp[3];
        const int64_t gx0 = floordiv(X0, bw), gx1 = floordiv(X1 - 1, bw) + 1;
        int64_t gy0 = floordiv(Y0, bh), gy1 = floordiv(Y1 - 1, bh) + 1;
        if (part_n > 0) {
            gy0 = std::max(gy0, lo_b);
            gy1 = std::min(gy1, hi_b);
            if (gy1 <= gy0) continue;
        }
        for (int64_t gy = gy0; gy < gy1; ++gy)
            for (int64_t gx = gx0; gx < gx1; ++gx) pairs.push_back({gy * nbx + gx, s, ids[s]});
        pw_max = std::max(pw_max, p->span_max(p->tables[t.tab_blend_h], bw, false));
        ph_max = std::max(ph_max, p->span_max(p->tables[t.tab_blend_v], bh, false));
        const double frac = part_n <= 0 ? 1.0 : (double)((gy1 - gy0) * bh) / (double)std::max(Y1 - Y0, (int64_t)1);
        nbytes += (int64_t)(std::min(frac, 1.0) * (double)(t.pw * t.ph * 3 * src_bytes + 2 * (sp[2] - sp[0]) * (sp[3] - sp[1]) * 3));
    }
    wl->path = path;
    wl->block_rows = bh;
    wl->block_cols = use_fast ? 0 : bw;
    if (pairs.empty()) {
        wl->item_words = use_fast ? USDU_JOB_WORDS : USDU_BLEND_ITEM_WORDS;
        wl->n_launch = 0;
        wl->patch_w = pw_max;
        wl->patch_h = ph_max;
        return USDU_OK;
    }
    // by block, then by position in the tile list (the order of the tile list IS the blend order)
    std::sort(pairs.begin(), pairs.end(), [](const Pair& a, const Pair& b) { return a.key != b.key ? a.key < b.key : a.seq < b.seq; });
    const size_t np = pairs.size();
    std::vector<size_t> first;
    for (size_t i = 0; i < np; ++i)
        if (i == 0 || pairs[i].key != pairs[i - 1].key) first.push_back(i);
    wl->algo_bytes = nbytes;
    wl->patch_w = pw_max;
    wl->patch_h = ph_max;
    if (!use_fast) {
        std::vector<int64_t> items(first.size() * USDU_BLEND_ITEM_WORDS), cover(np * USDU_COVER_WORDS, 0);
        for (size_t b = 0; b < first.size(); ++b) {
            const size_t e = b + 1 < first.size() ? first[b + 1] : np;
            items[4 * b + 0] = (pairs[first[b]].key % nbx) * bw;
            items[4 * b + 1] = (pairs[first[b]].key / nbx) * bh;
            items[4 * b + 2] = (int64_t)first[b];
            items[4 * b + 3] = (int64_t)(e - first[b]);
        }
        for (size_t i = 0; i < np; ++i) {
            const int64_t o = offs[pairs[i].seq];
            cover[4 * i + 0] = pairs[i].tid;
            cover[4 * i + 1] = o & 0xFFFFFFFF;
            cover[4 * i + 2] = o >> 32;
        }
        store_rows(wl->items, items);
        store_rows(wl->cover, cover);
        wl->item_words = USDU_BLEND_ITEM_WORDS;
        wl->n_launch = -1;
        return USDU_OK;
    }
    // (block, tile) pairs -> job records; the first record of every block comes first (they form the grid), the rest is
    // chained through USDU_J_NEXT
    const bool mma = path == 2;
    std::vector<int64_t> J(np * USDU_JOB_WORDS, 0);
    int64_t cols_max = INT64_MIN, need_w_max = INT64_MIN, rows_max = INT64_MIN, need_h_max = INT64_MIN;
    for (size_t i = 0; i < np; ++i) {
        const Pair& q = pairs[i];
        const Tile& t = p->tiles[q.tid];
        const Table& th_ = p->tables[t.tab_blend_h];
        const Table& tv = p->tables[t.tab_blend_v];
        const int32_t* desc = p->desc.data() + q.tid * USDU_TILE_WORDS;
        const int64_t bx0 = (q.key % nbx) * bw, by0 = (q.key / nbx) * bh;
        const int64_t ox_base = bx0 - t.x1, oy_base = by0 - t.y1;
        int64_t ix0, ix1, iy0, iy1, rows_h, rows_v, taps_h, taps_v;
        if (mma) {
            const MmaAxis ah = mma_axis(th_, ox_base, bw), av = mma_axis(tv, oy_base, bh);
            rows_h = ah.frag; taps_h = ah.ks; ix0 = ah.s0; ix1 = ix0 + ((ah.count + 3) & ~(int64_t)3);
            rows_v = av.frag; taps_v = av.ks; iy0 = av.s0; iy1 = iy0 + av.count;
            cols_max = std::max(cols_max, ix1 - ix0); need_w_max = std::max(need_w_max, ah.need);
            rows_max = std::max(rows_max, iy1 - iy0); need_h_max = std::max(need_h_max, av.need);
        } else {
            ix0 = first_of(th_, ox_base);
            ix1 = std::min(first_of(th_, ox_base + bw - 1) + th_.taps, (int64_t)th_.n_in);
            iy0 = first_of(tv, oy_base);
            iy1 = std::min(first_of(tv, oy_base + bh - 1) + tv.taps, (int64_t)tv.n_in);
            rows_h = th_.packed; taps_h = th_.job_taps;
            rows_v = tv.packed; taps_v = tv.job_taps;
        }
        const int64_t lead = mma ? 0 : (ix0 & 3);
        int64_t* r = &J[i * USDU_JOB_WORDS];
        r[USDU_J_TAPS_H] = taps_h; r[USDU_J_TAPS_V] = taps_v;
        const int64_t src = offs[q.seq] + (iy0 * t.pw + ix0 - lead) * 3;
        r[USDU_J_SRC_A] = src & 0xFFFFFFFF; r[USDU_J_SRC_B] = src >> 32; r[USDU_J_LEAD] = lead;
        r[USDU_J_COLS] = ix1 - ix0; r[USDU_J_ROWS] = iy1 - iy0; r[USDU_J_IX0] = ix0; r[USDU_J_IY0] = iy0;
        r[USDU_J_ROWS_H] = rows_h; r[USDU_J_OX_BASE] = ox_base; r[USDU_J_N_OUT_H] = t.ew();
        r[USDU_J_ROWS_V] = rows_v; r[USDU_J_OY_BASE] = oy_base; r[USDU_J_N_OUT_V] = t.eh();
        r[USDU_J_DST_X] = bx0; r[USDU_J_DST_Y] = by0;
        const int64_t mpitch = desc[USDU_T_MASK_PITCH];
        const int64_t moff = (int64_t)desc[USDU_T_MASK_OFF] + oy_base * mpitch + ox_base;          // may be negative
        r[USDU_J_OFF_LO] = moff & 0xFFFFFFFF; r[USDU_J_OFF_HI] = moff >> 32;
        const int64_t cw = std::min(bw, W - bx0), chh = std::min(bh, H - by0);
        const int64_t X0 = std::max(bx0, t.x1 + desc[USDU_T_SUP_X0]), X1 = std::min(bx0 + cw, t.x1 + desc[USDU_T_SUP_X1]);
        const int64_t Y0 = std::max(by0, t.y1 + desc[USDU_T_SUP_Y0]), Y1 = std::min(by0 + chh, t.y1 + desc[USDU_T_SUP_Y1]);
        r[USDU_J_CX0] = X0 - bx0; r[USDU_J_CX1] = X1 - bx0; r[USDU_J_CY0] = Y0 - by0; r[USDU_J_CY1] = Y1 - by0;
        r[USDU_J_ROWS_OUT] = Y1 - by0;
        const bool opaque = cw == bw && chh == bh && bx0 >= t.x1 + desc[USDU_T_FULL_X0] && bx0 + bw <= t.x1 + desc[USDU_T_FULL_X1] &&
                            by0 >= t.y1 + desc[USDU_T_FULL_Y0] && by0 + bh <= t.y1 + desc[USDU_T_FULL_Y1];
        r[USDU_J_FLAGS] = opaque ? 1 : 0;
        r[USDU_J_MPITCH] = mpitch;
        set_frame(r, t.pw, t.ph);
    }
    // record order: heads (one per block) first, then the rest; chain through NEXT
    std::vector<int64_t> pos(np);
    {
        size_t h = 0, rest = first.size(), f = 0;
        for (size_t i = 0; i < np; ++i) {
            const bool head = f < first.size() && first[f] == i;
            if (head) ++f;
            pos[i] = head ? (int64_t)h++ : (int64_t)rest++;
        }
    }
    std::vector<int64_t> out(np * USDU_JOB_WORDS);
    for (size_t i = 0; i < np; ++i) {
        J[i * USDU_JOB_WORDS + USDU_J_NEXT] = (i + 1 < np && pairs[i + 1].key == pairs[i].key) ? pos[i + 1] : -1;
        std::copy(&J[i * USDU_JOB_WORDS], &J[i * USDU_JOB_WORDS] + USDU_JOB_WORDS, &out[pos[i] * USDU_JOB_WORDS]);
    }
    if (mma) {
        wl->patch_w = std::max(cols_max, need_w_max);
        wl->patch_h = mma_patch_h(rows_max, need_h_max, wl->patch_w);
    }
    store_rows(wl->items, out);
    wl->item_words = USDU_JOB_WORDS;
    wl->n_launch = (int64_t)first.size();
    wl->ks2 = mma && any_ks2(wl->items);
    return USDU_OK;
}

// Does job record r stage a canvas pixel that the blend of a tile in prev[0..n_prev) changes (its feather support)?
bool meets(const Plan* p, const int32_t* r, const int32_t* prev, int n_prev) {
    const int64_t x0 = r[USDU_J_SRC_A], y0 = r[USDU_J_SRC_B];
    const int64_t x1 = x0 + r[USDU_J_LEAD] + r[USDU_J_COLS], y1 = y0 + r[USDU_J_ROWS];   // (integer-pipe records start `lead` pixels early)
    for (int i = 0; i < n_prev; ++i) {
        const Tile& t = p->tiles[prev[i]];
        int64_t s[4];
        p->support(t, s);
        if (s[2] > s[0] && s[3] > s[1] && x0 < t.x1 + s[2] && t.x1 + s[0] < x1 && y0 < t.y1 + s[3] && t.y1 + s[1] < y1) return true;
    }
    return false;
}

int64_t job_outputs(const int32_t* r) { return (int64_t)r[USDU_J_ROWS_OUT] * r[USDU_J_COLS_OUT]; }

// The jobs `pick` of crop lists (each entry: list, record index) as one launch: the layout of `shape`, patch words that
// hold every job's staging, algorithmic bytes by share of the outputs.
void take_jobs(const std::vector<std::pair<const WorkList*, size_t>>& pick, const WorkList& shape, int64_t all_outputs,
               WorkList* wl) {
    *wl = shape;
    wl->items.clear();
    int64_t outputs = 0, plane = shape.patch_h & 0xFFFF, mid = shape.patch_h >> 16;
    for (const auto& q : pick) {
        const int32_t* r = q.first->items.data() + q.second * USDU_JOB_WORDS;
        wl->items.insert(wl->items.end(), r, r + USDU_JOB_WORDS);
        outputs += job_outputs(r);
        wl->patch_w = std::max(wl->patch_w, q.first->patch_w);
        plane = std::max(plane, q.first->patch_h & 0xFFFF);
        mid = std::max(mid, q.first->patch_h >> 16);
    }
    if (shape.path == 2) wl->patch_h = plane | (mid << 16);
    wl->algo_bytes = (int64_t)((double)shape.algo_bytes * (double)outputs / (double)std::max(all_outputs, (int64_t)1));
    wl->ks2 = shape.path == 2 && any_ks2(wl->items);
}

int split_worklists(Plan* p, const int32_t* ids, const int64_t* offs, int n, const int32_t* prev, int n_prev, int B,
                    int req_path, const LaunchModel& m, WorkList* late, WorkList* early, WorkList* blend) {
    const int path = kernel_path(p, req_path);
    if (path < 1) {
        usdu::set_error("usdu_plan_split_worklists: this plan has no job-record kernels");
        return USDU_ERR_UNSUPPORTED;
    }
    WorkList shorts, talls;
    int s = crop_worklist(p, ids, n, B, path, LaunchModel{m.sm_count, path == 2 ? 16 : 0}, &shorts);
    if (s == USDU_OK && path == 2) s = crop_worklist(p, ids, n, B, path, LaunchModel{m.sm_count, 32}, &talls);
    if (s != USDU_OK) return s;
    const WorkList& tall = path == 2 ? talls : shorts;
    // short jobs by (output slot, column, first row): the short jobs inside a tall job's rows
    std::map<std::array<int64_t, 3>, size_t> short_at;
    int64_t all_outputs = 0;
    for (size_t j = 0; j < (size_t)shorts.n_items(); ++j) {
        const int32_t* r = shorts.items.data() + j * USDU_JOB_WORDS;
        short_at[{(int64_t)(uint32_t)r[USDU_J_OFF_LO] | (int64_t)r[USDU_J_OFF_HI] << 32, r[USDU_J_OX_BASE], r[USDU_J_OY_BASE]}] = j;
        all_outputs += job_outputs(r);
    }
    std::vector<std::pair<const WorkList*, size_t>> lj, ej;
    if (n_prev == 0) {
        for (size_t j = 0; j < (size_t)shorts.n_items(); ++j) lj.emplace_back(&shorts, j);
    } else {
        for (size_t j = 0; j < (size_t)tall.n_items(); ++j) {
            const int32_t* r = tall.items.data() + j * USDU_JOB_WORDS;
            if (!meets(p, r, prev, n_prev)) {
                ej.emplace_back(&tall, j);
                continue;
            }
            const int64_t slot = (int64_t)(uint32_t)r[USDU_J_OFF_LO] | (int64_t)r[USDU_J_OFF_HI] << 32;
            int64_t covered = 0;
            for (auto it = short_at.lower_bound({slot, r[USDU_J_OX_BASE], r[USDU_J_OY_BASE]});
                 it != short_at.end() && it->first[0] == slot && it->first[1] == r[USDU_J_OX_BASE] &&
                 it->first[2] < (int64_t)r[USDU_J_OY_BASE] + r[USDU_J_ROWS_OUT];
                 ++it) {
                const int32_t* q = shorts.items.data() + it->second * USDU_JOB_WORDS;
                (meets(p, q, prev, n_prev) ? lj : ej).emplace_back(&shorts, it->second);
                covered += job_outputs(q);
            }
            if (covered != job_outputs(r)) {
                usdu::set_error("usdu_plan_split_worklists: the short jobs of a tall crop job cover %lld of its %lld outputs",
                                (long long)covered, (long long)job_outputs(r));
                return USDU_ERR_INVALID;
            }
        }
    }
    take_jobs(lj, shorts, all_outputs, late);
    take_jobs(ej, tall, all_outputs, early);
    int64_t outputs = 0;
    for (const WorkList* wl : {late, early})
        for (size_t j = 0; j < (size_t)wl->n_items(); ++j) outputs += job_outputs(wl->items.data() + j * USDU_JOB_WORDS);
    if (outputs != all_outputs) {
        usdu::set_error("usdu_plan_split_worklists: early and late jobs cover %lld of %lld outputs", (long long)outputs,
                        (long long)all_outputs);
        return USDU_ERR_INVALID;
    }
    if (path != 2) return blend_worklist(p, ids, offs, n, 4, B, path, 0, 0, m, blend);
    // blend: cost(bh) = ceil(CTAs / resident slots) * (staged rows + written rows) per CTA
    const int sms = m.sm_count > 0 ? m.sm_count : (usdu::sm_count() > 0 ? usdu::sm_count() : kDefaultSms);
    const bool device = m.sm_count == 0 && usdu::sm_count() > 0;
    int64_t best_cost = -1;
    for (int bh : {32, 16}) {
        WorkList wl;
        if ((s = blend_worklist(p, ids, offs, n, 4, B, path, 0, 0, LaunchModel{m.sm_count, bh}, &wl)) != USDU_OK) return s;
        if (wl.n_launch <= 0) {
            *blend = std::move(wl);
            return USDU_OK;
        }
        const int per_sm = usdu::mma::resident_ctas(USDU_KERNEL_BLEND, wl.ks2, (int)wl.patch_w, (int)wl.patch_h, bh, device);
        if (per_sm < 0) return per_sm;
        const int64_t slots = (int64_t)sms * std::max(per_sm, 1);
        const int64_t cost = ceildiv(wl.n_launch * B, slots) * ((wl.patch_h & 0xFFFF) + bh);
        if (best_cost < 0 || cost < best_cost) {
            best_cost = cost;
            *blend = std::move(wl);
        }
    }
    return USDU_OK;
}

template <class F>
int guarded(F&& f) {
    try {
        return f();
    } catch (const std::bad_alloc&) {
        usdu::set_error("out of host memory");
        return USDU_ERR_INVALID;
    }
}

}  // namespace

extern "C" {

int64_t usdu_canvas_pitch(int W) {
    if (W <= 0) {
        usdu::set_error("usdu_canvas_pitch: width must be positive (%d)", W);
        return USDU_ERR_INVALID;
    }
    return ((int64_t)W * 3 + 127) / 128 * 128;
}

int64_t usdu_canvas_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) {
        usdu::set_error("usdu_canvas_bytes: sizes must be positive (B=%d H=%d W=%d)", B, H, W);
        return USDU_ERR_INVALID;
    }
    return (int64_t)B * H * usdu_canvas_pitch(W) + USDU_CANVAS_SLACK;
}

int usdu_plan_create(int W, int H, int tile_width, int tile_height, int padding, int mask_blur, int uniform, usdu_plan** plan) {
    if (!plan) {
        usdu::set_error("usdu_plan_create: plan is null");
        return USDU_ERR_INVALID;
    }
    *plan = nullptr;
    return guarded([&]() {
        Plan* p = new Plan();
        p->W = W; p->H = H; p->tile_width = tile_width; p->tile_height = tile_height;
        p->padding = padding; p->mask_blur = mask_blur; p->uniform = uniform != 0;
        int s;
        try {
            s = build_plan(p);
        } catch (...) {
            delete p;
            throw;
        }
        if (s != USDU_OK) {
            delete p;
            return s;
        }
        *plan = reinterpret_cast<usdu_plan*>(p);
        return (int)USDU_OK;
    });
}

int usdu_plan_destroy(usdu_plan* plan) {
    delete reinterpret_cast<Plan*>(plan);
    return USDU_OK;
}

#define USDU_PLAN_ARG(p)                                       \
    do {                                                       \
        if (!(p)) {                                            \
            usdu::set_error("%s: plan is null", __func__);     \
            return USDU_ERR_INVALID;                           \
        }                                                      \
    } while (0)

int usdu_plan_info(const usdu_plan* plan, int64_t* info) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    if (!info) {
        usdu::set_error("usdu_plan_info: info is null");
        return USDU_ERR_INVALID;
    }
    for (int i = 0; i < USDU_PLAN_INFO_WORDS; ++i) info[i] = 0;
    info[USDU_PI_TW] = p->tw;
    info[USDU_PI_TH] = p->th;
    info[USDU_PI_TILES] = (int64_t)p->tiles.size();
    info[USDU_PI_TAB_WORDS] = (int64_t)p->tabs.size();
    info[USDU_PI_TABLES] = (int64_t)p->tables.size();
    info[USDU_PI_MASK_CLASSES] = (int64_t)(p->specs.size() / USDU_MASK_WORDS);
    info[USDU_PI_MASK_POOL_BYTES] = p->mask_pool_bytes;
    info[USDU_PI_FAST] = p->fast;
    info[USDU_PI_MMA] = p->mma;
    info[USDU_PI_PATH] = kernel_path(p, 2);
    int64_t nb = 0;
    for (const auto& v : p->neighbors) nb += (int64_t)v.size();
    info[USDU_PI_NEIGHBOR_WORDS] = nb;
    return USDU_OK;
}

#define USDU_OUT_ARG(ptr)                                      \
    do {                                                       \
        if (!(ptr)) {                                          \
            usdu::set_error("%s: output array is null", __func__); \
            return USDU_ERR_INVALID;                           \
        }                                                      \
    } while (0)

int usdu_plan_tiles(const usdu_plan* plan, int32_t* tiles) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    USDU_OUT_ARG(tiles);
    for (size_t i = 0; i < p->tiles.size(); ++i) {
        const Tile& t = p->tiles[i];
        const int64_t w[USDU_PLAN_TILE_WORDS] = {t.x, t.y, t.x1, t.y1, t.ew(), t.eh(), t.pw, t.ph, t.bx2, t.by2, p->mask_class[i], 0};
        for (int k = 0; k < USDU_PLAN_TILE_WORDS; ++k) tiles[i * USDU_PLAN_TILE_WORDS + k] = (int32_t)w[k];
    }
    return USDU_OK;
}

int usdu_plan_tile_desc(const usdu_plan* plan, int32_t* desc) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    USDU_OUT_ARG(desc);
    if (!p->desc.empty()) memcpy(desc, p->desc.data(), p->desc.size() * sizeof(int32_t));
    return USDU_OK;
}

int usdu_plan_tables(const usdu_plan* plan, int32_t* pool) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    USDU_OUT_ARG(pool);
    if (!p->tabs.empty()) memcpy(pool, p->tabs.data(), p->tabs.size() * sizeof(int32_t));
    return USDU_OK;
}

int usdu_plan_table_index(const usdu_plan* plan, int32_t* index) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    USDU_OUT_ARG(index);
    for (size_t i = 0; i < p->tables.size(); ++i) {
        const Table& tb = p->tables[i];
        const int64_t w[USDU_PLAN_TABLE_WORDS] = {tb.n_in, tb.n_out, tb.off, tb.packed, tb.frag, tb.ks, tb.taps, tb.job_taps};
        for (int k = 0; k < USDU_PLAN_TABLE_WORDS; ++k) index[i * USDU_PLAN_TABLE_WORDS + k] = (int32_t)w[k];
    }
    return USDU_OK;
}

int usdu_plan_mask_specs(const usdu_plan* plan, int32_t* specs) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    USDU_OUT_ARG(specs);
    if (!p->specs.empty()) memcpy(specs, p->specs.data(), p->specs.size() * sizeof(int32_t));
    return USDU_OK;
}

int usdu_plan_neighbors(const usdu_plan* plan, int32_t* first, int32_t* list) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    USDU_OUT_ARG(first);
    int64_t k = 0;
    for (size_t i = 0; i < p->neighbors.size(); ++i) {
        first[i] = (int32_t)k;
        for (int j : p->neighbors[i]) {
            USDU_OUT_ARG(list);
            list[k++] = j;
        }
    }
    first[p->neighbors.size()] = (int32_t)k;
    return USDU_OK;
}

int usdu_plan_waves(const usdu_plan* plan, const int32_t* order, int n, int32_t* wave) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    const int s = check_ids(p, order, n, "usdu_plan_waves");
    if (s != USDU_OK) return s;
    if (n > 0 && !wave) {
        usdu::set_error("usdu_plan_waves: wave is null");
        return USDU_ERR_INVALID;
    }
    return guarded([&]() {
        std::vector<int64_t> pos(p->tiles.size(), -1);
        for (int i = 0; i < n; ++i) {
            if (pos[order[i]] >= 0) {
                usdu::set_error("usdu_plan_waves: tile %d appears twice in the order", order[i]);
                return (int)USDU_ERR_INVALID;
            }
            pos[order[i]] = i;
        }
        // tile k must see the blends of every earlier tile whose window intersects its own
        std::vector<int32_t> level(p->tiles.size(), 0);
        int n_waves = 0;
        for (int i = 0; i < n; ++i) {
            const int t = order[i];
            int lv = 0;
            for (int nb : p->neighbors[t])
                if (pos[nb] >= 0 && pos[nb] < i) lv = std::max(lv, level[nb] + 1);
            level[t] = lv;
            wave[i] = lv;
            n_waves = std::max(n_waves, lv + 1);
        }
        return n_waves;
    });
}

int usdu_plan_crop_worklist(const usdu_plan* plan, const int32_t* tile_ids, int n, int B, int path, int sm_count,
                            int mma_block_rows, usdu_worklist** wl) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    if (!wl) {
        usdu::set_error("usdu_plan_crop_worklist: wl is null");
        return USDU_ERR_INVALID;
    }
    *wl = nullptr;
    int s = check_ids(p, tile_ids, n, "usdu_plan_crop_worklist");
    if (s != USDU_OK) return s;
    if (B <= 0 || path < 0 || sm_count < 0 || mma_block_rows < 0 || mma_block_rows > USDU_FAST_BLOCK_H) {
        usdu::set_error("usdu_plan_crop_worklist: bad arguments (B=%d path=%d sm_count=%d mma_block_rows=%d)", B, path, sm_count, mma_block_rows);
        return USDU_ERR_INVALID;
    }
    return guarded([&]() {
        WorkList* w = new WorkList();
        // the plan caches its generic block shape: a pure function of the plan
        const int r = crop_worklist(const_cast<Plan*>(p), tile_ids, n, B, path, LaunchModel{sm_count, mma_block_rows}, w);
        if (r != USDU_OK) {
            delete w;
            return r;
        }
        *wl = reinterpret_cast<usdu_worklist*>(w);
        return (int)USDU_OK;
    });
}

int usdu_plan_blend_worklist(const usdu_plan* plan, const int32_t* tile_ids, const int64_t* src_offsets, int n, int src_bytes,
                             int B, int path, int part_i, int part_n, int sm_count, int mma_block_rows, usdu_worklist** wl) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    if (!wl) {
        usdu::set_error("usdu_plan_blend_worklist: wl is null");
        return USDU_ERR_INVALID;
    }
    *wl = nullptr;
    int s = check_ids(p, tile_ids, n, "usdu_plan_blend_worklist");
    if (s != USDU_OK) return s;
    if ((n > 0 && !src_offsets) || (src_bytes != 1 && src_bytes != 4) || B <= 0 || path < 0 || part_n < 0 ||
        (part_n > 0 && (part_i < 0 || part_i >= part_n)) || sm_count < 0 || mma_block_rows < 0 ||
        mma_block_rows > USDU_FAST_BLOCK_H) {
        usdu::set_error("usdu_plan_blend_worklist: bad arguments (src_bytes=%d B=%d path=%d part=%d/%d sm_count=%d "
                        "mma_block_rows=%d)", src_bytes, B, path, part_i, part_n, sm_count, mma_block_rows);
        return USDU_ERR_INVALID;
    }
    return guarded([&]() {
        WorkList* w = new WorkList();
        const int r = blend_worklist(const_cast<Plan*>(p), tile_ids, src_offsets, n, src_bytes, B, path, part_i, part_n,
                                     LaunchModel{sm_count, mma_block_rows}, w);
        if (r != USDU_OK) {
            delete w;
            return r;
        }
        *wl = reinterpret_cast<usdu_worklist*>(w);
        return (int)USDU_OK;
    });
}

int usdu_plan_split_worklists(const usdu_plan* plan, const int32_t* tile_ids, const int64_t* src_offsets, int n,
                              const int32_t* prev_ids, int n_prev, int B, int path, int sm_count, usdu_worklist** late,
                              usdu_worklist** early, usdu_worklist** blend) {
    const Plan* p = reinterpret_cast<const Plan*>(plan);
    USDU_PLAN_ARG(p);
    if (!late || !early || !blend) {
        usdu::set_error("usdu_plan_split_worklists: an output handle is null");
        return USDU_ERR_INVALID;
    }
    *late = *early = *blend = nullptr;
    int s = check_ids(p, tile_ids, n, "usdu_plan_split_worklists");
    if (s == USDU_OK) s = check_ids(p, prev_ids, n_prev, "usdu_plan_split_worklists (previous wave)");
    if (s != USDU_OK) return s;
    if ((n > 0 && !src_offsets) || B <= 0 || path < 1 || sm_count < 0) {
        usdu::set_error("usdu_plan_split_worklists: bad arguments (B=%d path=%d sm_count=%d)", B, path, sm_count);
        return USDU_ERR_INVALID;
    }
    return guarded([&]() {
        WorkList *l = new WorkList(), *e = new WorkList(), *b = new WorkList();
        const int r = split_worklists(const_cast<Plan*>(p), tile_ids, src_offsets, n, prev_ids, n_prev, B, path,
                                      LaunchModel{sm_count, 0}, l, e, b);
        if (r != USDU_OK) {
            delete l;
            delete e;
            delete b;
            return r;
        }
        *late = reinterpret_cast<usdu_worklist*>(l);
        *early = reinterpret_cast<usdu_worklist*>(e);
        *blend = reinterpret_cast<usdu_worklist*>(b);
        return (int)USDU_OK;
    });
}

int usdu_worklist_destroy(usdu_worklist* wl) {
    delete reinterpret_cast<WorkList*>(wl);
    return USDU_OK;
}

int usdu_worklist_info(const usdu_worklist* handle, int64_t* info) {
    const WorkList* wl = reinterpret_cast<const WorkList*>(handle);
    if (!wl || !info) {
        usdu::set_error("usdu_worklist_info: null argument");
        return USDU_ERR_INVALID;
    }
    for (int i = 0; i < USDU_WL_INFO_WORDS; ++i) info[i] = 0;
    static const int path_flags[3] = {0, USDU_FLAG_FAST, USDU_FLAG_MMA};
    info[USDU_WL_ITEMS] = wl->n_items();
    info[USDU_WL_ITEM_WORDS] = wl->item_words;
    info[USDU_WL_COVER] = (int64_t)(wl->cover.size() / USDU_COVER_WORDS);
    info[USDU_WL_PATCH_W] = wl->patch_w;
    info[USDU_WL_PATCH_H] = wl->patch_h;
    info[USDU_WL_ALGO_BYTES] = wl->algo_bytes;
    info[USDU_WL_N_LAUNCH] = wl->n_launch;
    info[USDU_WL_BLOCK_ROWS] = wl->block_rows;
    info[USDU_WL_BLOCK_COLS] = wl->block_cols;
    info[USDU_WL_ROW0] = wl->row0;
    info[USDU_WL_ROW1] = wl->row1;
    info[USDU_WL_PATH] = wl->path;
    info[USDU_WL_KS2] = wl->ks2;
    info[USDU_WL_TOTAL] = wl->total;
    info[USDU_WL_FLAGS] = path_flags[wl->path] | (wl->block_rows << 8) | (wl->block_cols << 16) | (wl->ks2 ? USDU_FLAG_MMA_KS2 : 0);
    info[USDU_WL_GRID] = wl->n_launch >= 0 ? wl->n_launch : wl->n_items();
    return USDU_OK;
}

int usdu_worklist_items(const usdu_worklist* handle, int32_t* items) {
    const WorkList* wl = reinterpret_cast<const WorkList*>(handle);
    if (!wl || !items) {
        usdu::set_error("usdu_worklist_items: null argument");
        return USDU_ERR_INVALID;
    }
    if (!wl->items.empty()) memcpy(items, wl->items.data(), wl->items.size() * sizeof(int32_t));
    return USDU_OK;
}

int usdu_worklist_cover(const usdu_worklist* handle, int32_t* cover) {
    const WorkList* wl = reinterpret_cast<const WorkList*>(handle);
    if (!wl || !cover) {
        usdu::set_error("usdu_worklist_cover: null argument");
        return USDU_ERR_INVALID;
    }
    if (!wl->cover.empty()) memcpy(cover, wl->cover.data(), wl->cover.size() * sizeof(int32_t));
    return USDU_OK;
}

int usdu_worklist_slots(const usdu_worklist* handle, int64_t* offsets) {
    const WorkList* wl = reinterpret_cast<const WorkList*>(handle);
    if (!wl || !offsets) {
        usdu::set_error("usdu_worklist_slots: null argument");
        return USDU_ERR_INVALID;
    }
    if (!wl->slots.empty()) memcpy(offsets, wl->slots.data(), wl->slots.size() * sizeof(int64_t));
    return USDU_OK;
}

}  // extern "C"
