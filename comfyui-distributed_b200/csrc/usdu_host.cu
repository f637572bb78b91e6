// usdu_host.cu -- library plumbing and the host-side table builders.
//
// The builders restate Pillow's setup arithmetic with the same C types Pillow uses so
// the fixed-point tables are bit-identical to what the reference's CPU path gets from
// Image.resize(..., LANCZOS) (upscale/tile_ops.py:88,148,329) and
// ImageFilter.GaussianBlur (upscale/tile_ops.py:306):
//   Resample.c  precompute_coeffs / normalize_coeffs_8bpc  -> usdu_build_resample_table
//   BoxBlur.c   _gaussian_blur_radius / ImagingHorizontalBoxBlur -> usdu_box_blur_params
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <atomic>
#include <vector>

#include "usdu_common.cuh"

namespace usdu {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return USDU_OK;
    set_error("CUDA error %d (%s) in %s", static_cast<int>(e), cudaGetErrorString(e), what);
    return USDU_ERR_CUDA;
}

int sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    const bool cached = e == cudaSuccess && dev >= 0 && dev < 64;
    if (cached) {
        const int c = cache[dev].load(std::memory_order_relaxed);
        if (c > 0) return c;
    }
    int n = 0;
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) {
        check_cuda(e, "cudaDeviceGetAttribute(cudaDevAttrMultiProcessorCount)");
        cudaGetLastError();
        return USDU_ERR_CUDA;
    }
    if (cached) cache[dev].store(n, std::memory_order_relaxed);
    return n;
}

}  // namespace usdu

extern "C" {

int usdu_abi_version(void) { return USDU_ABI_VERSION; }

const char* usdu_last_error(void) { return usdu::g_err; }

int usdu_sm_count(void) { return usdu::sm_count(); }

int usdu_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        usdu::check_cuda(e, "cudaGetDeviceCount");
        cudaGetLastError();
        return USDU_ERR_CUDA;
    }
    return n;
}

// ---- LANCZOS tables -------------------------------------------------------------------
static double sinc_filter(double x) {
    if (x == 0.0) return 1.0;
    x = x * M_PI;
    return sin(x) / x;
}

static double lanczos_filter(double x) {
    /* truncated sinc, support 3 */
    if (-3.0 <= x && x < 3.0) return sinc_filter(x) * sinc_filter(x / 3);
    return 0.0;
}

static double bicubic_filter(double x) {
    /* Keys cubic, a = -0.5, support 2 (Resample.c bicubic_filter; utils/usdu_utils.py:424,435) */
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}

static double filter_support(int filter) { return filter == USDU_FILTER_BICUBIC ? 2.0 : 3.0; }

int usdu_filter_ksize(int filter, int in_size, int out_size) {
    if (in_size <= 0 || out_size <= 0) {
        usdu::set_error("usdu_filter_ksize: sizes must be positive (%d -> %d)", in_size, out_size);
        return USDU_ERR_INVALID;
    }
    if (filter != USDU_FILTER_LANCZOS && filter != USDU_FILTER_BICUBIC) {
        usdu::set_error("usdu_filter_ksize: unknown filter %d", filter);
        return USDU_ERR_INVALID;
    }
    double filterscale = (double)in_size / out_size;
    if (filterscale < 1.0) filterscale = 1.0;
    double support = filter_support(filter) * filterscale;
    return (int)ceil(support) * 2 + 1;
}

int usdu_resample_ksize(int in_size, int out_size) { return usdu_filter_ksize(USDU_FILTER_LANCZOS, in_size, out_size); }

int64_t usdu_filter_table_words(int filter, int in_size, int out_size) {
    int ks = usdu_filter_ksize(filter, in_size, out_size);
    if (ks < 0) return ks;
    // the packed rows are read with 128-bit loads: their start is padded to 4 int32
    return (((int64_t)USDU_TAB_HEADER + (int64_t)out_size * (2 + ks) + 3) & ~(int64_t)3) + (int64_t)out_size * 2 * USDU_PACKED_ROW;
}

int64_t usdu_resample_table_words(int in_size, int out_size) {
    return usdu_filter_table_words(USDU_FILTER_LANCZOS, in_size, out_size);
}

int usdu_build_resample_table(int in_size, int out_size, int32_t* table) {
    return usdu_build_filter_table(USDU_FILTER_LANCZOS, in_size, out_size, table);
}

int usdu_build_filter_table(int filter, int in_size, int out_size, int32_t* table) {
    USDU_REQUIRE(table != nullptr, "usdu_build_filter_table: table is null");
    int ksize = usdu_filter_ksize(filter, in_size, out_size);
    if (ksize < 0) return ksize;
    double (*const weight)(double) = filter == USDU_FILTER_BICUBIC ? bicubic_filter : lanczos_filter;
    double scale, filterscale;
    scale = filterscale = (double)in_size / out_size;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = filter_support(filter) * filterscale;
    const double ss = 1.0 / filterscale;
    table[0] = in_size;
    table[1] = out_size;
    table[2] = ksize;
    for (int i = 3; i < USDU_TAB_HEADER; ++i) table[i] = 0;
    int32_t* bounds = table + USDU_TAB_HEADER;
    int32_t* kk = bounds + 2 * (int64_t)out_size;
    std::vector<double> w(ksize);
    for (int xx = 0; xx < out_size; xx++) {
        double center = (xx + 0.5) * scale;
        double ww = 0.0;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        for (int x = 0; x < xmax; x++) {
            double v = weight((x + xmin - center + 0.5) * ss);
            w[x] = v;
            ww += v;
        }
        int32_t* k = kk + (int64_t)xx * ksize;
        for (int x = 0; x < xmax; x++) {
            double v = w[x];
            if (ww != 0.0) v /= ww;
            if (v < 0)
                k[x] = (int)(-0.5 + v * (1 << usdu::kPrecisionBits));
            else
                k[x] = (int)(0.5 + v * (1 << usdu::kPrecisionBits));
        }
        for (int x = xmax; x < ksize; x++) k[x] = 0;
        bounds[xx * 2 + 0] = xmin;
        bounds[xx * 2 + 1] = xmax;
    }
    // Packed rows for the fast kernels: {first input index, k0..k6}, usable when no output
    // needs more than USDU_FAST_TAPS taps and any USDU_FAST_GROUP consecutive outputs read at
    // most USDU_FAST_WINDOW consecutive inputs.
    int32_t* packed = table + (((int64_t)USDU_TAB_HEADER + (int64_t)out_size * (2 + ksize) + 3) & ~(int64_t)3);
    for (int32_t* q = kk + (int64_t)out_size * ksize; q < packed; ++q) *q = 0;
    int tmax = 0, span = 0;
    for (int xx = 0; xx < out_size; xx++) {
        if (bounds[xx * 2 + 1] > tmax) tmax = bounds[xx * 2 + 1];
        int last = xx + USDU_FAST_GROUP - 1 < out_size ? xx + USDU_FAST_GROUP - 1 : out_size - 1;
        int sp = bounds[last * 2] + USDU_FAST_TAPS - bounds[xx * 2];
        if (sp > span) span = sp;
    }
    table[3] = tmax;
    table[5] = span;
    const bool fast = tmax <= USDU_FAST_TAPS_WIDE;
    const int stride = tmax <= USDU_FAST_TAPS ? USDU_PACKED_ROW : 2 * USDU_PACKED_ROW;
    table[4] = fast ? (int32_t)(packed - table) : 0;
    table[6] = stride;
    for (int xx = 0; xx < out_size; xx++) {
        int32_t* r = packed + (int64_t)xx * stride;
        r[0] = bounds[xx * 2];
        for (int t = 0; t < stride - 1; ++t)
            r[1 + t] = (fast && t < bounds[xx * 2 + 1]) ? kk[(int64_t)xx * ksize + t] : 0;
    }
    return USDU_OK;
}

int usdu_build_identity_table(int size, int32_t* table) {
    USDU_REQUIRE(table != nullptr && size > 0, "usdu_build_identity_table: bad arguments");
    // Pillow skips a pass whose axis keeps its size (Resample.c ImagingResampleInner); one tap
    // of weight 2^22 reproduces that exactly: (v * 2^22 + 2^21) >> 22 == v.
    table[0] = size; table[1] = size; table[2] = 1; table[3] = 1;
    table[4] = (USDU_TAB_HEADER + 3 * size + 3) & ~3; table[5] = USDU_FAST_GROUP - 1 + USDU_FAST_TAPS; table[6] = USDU_PACKED_ROW; table[7] = 0;
    int32_t* bounds = table + USDU_TAB_HEADER;
    int32_t* kk = bounds + 2 * (int64_t)size;
    int32_t* packed = table + table[4];
    for (int32_t* q = kk + size; q < packed; ++q) *q = 0;
    for (int i = 0; i < size; ++i) {
        bounds[2 * i] = i; bounds[2 * i + 1] = 1; kk[i] = 1 << usdu::kPrecisionBits;
        int32_t* r = packed + (int64_t)i * USDU_PACKED_ROW;
        r[0] = i; r[1] = 1 << usdu::kPrecisionBits;
        for (int t = 1; t < USDU_FAST_TAPS; ++t) r[1 + t] = 0;
    }
    return USDU_OK;
}

// ---- Image.resize(..., NEAREST) source indices -------------------------------------
int usdu_nearest_index(int in_size, int out_size, int32_t* index) {
    USDU_REQUIRE(index != nullptr && in_size > 0 && out_size > 0, "usdu_nearest_index: bad arguments (%d -> %d)", in_size, out_size);
    // Geometry.c ImagingScaleAffine: xo = a/2, then xo += a per sample (the additions accumulate
    // in double exactly like the C loop), index = (int)xo.  utils/usdu_utils.py:190-199 stretches
    // the edge strips of pad_image2 this way.
    const double a = (double)in_size / out_size;
    double xo = 0.0 + a * 0.5;
    for (int x = 0; x < out_size; ++x) {
        int xin = xo < 0.0 ? -1 : (int)xo;
        if (xin < 0) xin = 0;
        if (xin > in_size - 1) xin = in_size - 1;
        index[x] = xin;
        xo += a;
    }
    return USDU_OK;
}

// ---- Gaussian-as-3-box parameters ---------------------------------------------------
int usdu_box_blur_params(float radius, int32_t* rad, uint32_t* ww, uint32_t* fw) {
    USDU_REQUIRE(rad && ww && fw, "usdu_box_blur_params: null output pointer");
    USDU_REQUIRE(radius > 0.0f, "usdu_box_blur_params: radius must be > 0");
    const float passes = 3;
    // volatile keeps every step a rounded C float exactly like BoxBlur.c compiled for x86-64
    volatile float sigma2 = radius * radius / passes;
    volatile float L = sqrt(12.0 * sigma2 + 1.0);
    volatile float l = floor((L - 1.0) / 2.0);
    volatile float a = (2 * l + 1) * (l * (l + 1) - 3 * sigma2);
    a = a / (6 * (sigma2 - (l + 1) * (l + 1)));
    volatile float fr = l + a;
    int r = (int)fr;
    uint32_t w = (uint32_t)((uint32_t)(1 << 24) / (fr * 2 + 1));
    uint32_t f = ((1 << 24) - (r * 2 + 1) * w) / 2;
    *rad = r;
    *ww = w;
    *fw = f;
    return USDU_OK;
}

}  // extern "C"
