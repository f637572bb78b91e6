// usdu_plane.cu -- one-channel u8 planes: the per-tile crop of conditioning masks.
//
// Reference: utils/usdu_utils.py:415-442 (crop_mask) -> per mask frame
//   tensor_to_pil -> resize(canvas, BICUBIC) -> crop(region) -> resize_and_pad_image(fill=True)
//   (:242-266: LANCZOS to the aspect-preserving size, pad_image2 edge fill :169-203, LANCZOS to
//   the tile size) -> BICUBIC if still not the tile size -> pil_to_tensor.
// All of it is Pillow 8bpc arithmetic on mode "L"; the kernels below evaluate the same
// fixed-point sums (Resample.c ImagingResampleHorizontal_8bpc / Vertical_8bpc) for the output
// WINDOW only, so the full-canvas BICUBIC upscale the reference does per tile and per frame
// (33 MP at 8K) becomes a crop-sized job.  HBM-bound byte work: 4 outputs per thread, 32-bit
// stores, coefficient tables read through L1.
#include "usdu_common.cuh"

namespace usdu {
namespace plane {

__device__ __forceinline__ uint32_t finish8(int acc) { return clip8(acc >> kPrecisionBits); }

struct PlaneView {
    const uint8_t* base;
    int64_t pitch, plane;
};

// ---- horizontal pass: out[p][r][i] for rows r0.. of the source, output columns ox.. ------------
__global__ void __launch_bounds__(kThreads)
hpass_kernel(PlaneView src, int n, int r0, int rows, const int32_t* __restrict__ tab, int ox, int ow,
             uint8_t* __restrict__ out, int64_t out_pitch, int64_t out_plane) {
    pdl_launch_dependents();
    const TableView t = table_at(tab, 0);
    const int quads = (ow + 3) >> 2;
    const int64_t total = (int64_t)n * rows * quads;
    pdl_wait();
    for (int64_t id = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; id < total; id += (int64_t)gridDim.x * blockDim.x) {
        const int q = (int)(id % quads);
        const int r = (int)((id / quads) % rows);
        const int p = (int)(id / ((int64_t)quads * rows));
        const uint8_t* line = src.base + p * src.plane + (int64_t)(r0 + r) * src.pitch;
        uint32_t word = 0;
        const int i0 = q * 4;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int i = i0 + e;
            if (i < ow) {
                const int xmin = t.bounds[2 * (ox + i)], cnt = t.bounds[2 * (ox + i) + 1];
                const int32_t* k = t.kk + (int64_t)(ox + i) * t.ksize;
                int acc = 1 << (kPrecisionBits - 1);
                for (int x = 0; x < cnt; ++x) acc += (int)line[xmin + x] * k[x];
                word |= finish8(acc) << (8 * e);
            }
        }
        uint8_t* o = out + p * out_plane + (int64_t)r * out_pitch + i0;
        if (i0 + 4 <= ow && ((reinterpret_cast<uintptr_t>(o) & 3) == 0)) {
            *reinterpret_cast<uint32_t*>(o) = word;
        } else {
            for (int e = 0; e < 4 && i0 + e < ow; ++e) o[e] = (uint8_t)(word >> (8 * e));
        }
    }
}

// ---- vertical pass: out[p][j][i] = sum over input rows of in[p][row - in_y0][in_x0 + i] --------
__global__ void __launch_bounds__(kThreads)
vpass_kernel(PlaneView in, int n, int in_y0, int in_x0, const int32_t* __restrict__ tab, int oy, int oh, int ow,
             uint8_t* __restrict__ out, int64_t out_pitch, int64_t out_plane) {
    pdl_launch_dependents();
    const TableView t = table_at(tab, 0);
    const int quads = (ow + 3) >> 2;
    const int64_t total = (int64_t)n * oh * quads;
    pdl_wait();
    for (int64_t id = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; id < total; id += (int64_t)gridDim.x * blockDim.x) {
        const int q = (int)(id % quads);
        const int j = (int)((id / quads) % oh);
        const int p = (int)(id / ((int64_t)quads * oh));
        const int ymin = t.bounds[2 * (oy + j)], cnt = t.bounds[2 * (oy + j) + 1];
        const int32_t* k = t.kk + (int64_t)(oy + j) * t.ksize;
        const int i0 = q * 4;
        const int lanes = min(4, ow - i0);
        int acc[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] = 1 << (kPrecisionBits - 1);
        const uint8_t* col = in.base + p * in.plane + (int64_t)(ymin - in_y0) * in.pitch + in_x0 + i0;
        const bool wide = lanes == 4 && ((reinterpret_cast<uintptr_t>(col) | (uintptr_t)in.pitch) & 3) == 0;
        for (int y = 0; y < cnt; ++y) {
            const int w = k[y];
            if (wide) {
                const uint32_t v = *reinterpret_cast<const uint32_t*>(col);
                acc[0] += (int)(v & 255u) * w;
                acc[1] += (int)((v >> 8) & 255u) * w;
                acc[2] += (int)((v >> 16) & 255u) * w;
                acc[3] += (int)(v >> 24) * w;
            } else {
                for (int e = 0; e < lanes; ++e) acc[e] += (int)col[e] * w;
            }
            col += in.pitch;
        }
        uint32_t word = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) word |= finish8(acc[e]) << (8 * e);
        uint8_t* o = out + p * out_plane + (int64_t)j * out_pitch + i0;
        if (lanes == 4 && ((reinterpret_cast<uintptr_t>(o) & 3) == 0)) {
            *reinterpret_cast<uint32_t*>(o) = word;
        } else {
            for (int e = 0; e < lanes; ++e) o[e] = (uint8_t)(word >> (8 * e));
        }
    }
}

// ---- window copy (both axes keep their size) ---------------------------------------------------
__global__ void __launch_bounds__(kThreads)
copy_kernel(PlaneView src, int n, int y0, int x0, int h, int w, uint8_t* __restrict__ out, int64_t out_pitch, int64_t out_plane) {
    pdl_launch_dependents();
    const int64_t total = (int64_t)n * h * w;
    pdl_wait();
    for (int64_t id = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; id < total; id += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(id % w);
        const int y = (int)((id / w) % h);
        const int p = (int)(id / ((int64_t)w * h));
        out[p * out_plane + (int64_t)y * out_pitch + x] = src.base[p * src.plane + (int64_t)(y0 + y) * src.pitch + x0 + x];
    }
}

// ---- pad_image2(fill=True) ----------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
pad_fill_kernel(PlaneView src, int n, int h, int w, int hp, int vp, const int32_t* __restrict__ row_index,
                const int32_t* __restrict__ col_index, uint8_t* __restrict__ out, int64_t out_pitch, int64_t out_plane) {
    pdl_launch_dependents();
    const int nh = h + 2 * vp, nw = w + 2 * hp;
    const int64_t total = (int64_t)n * nh * nw;
    pdl_wait();
    for (int64_t id = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; id < total; id += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(id % nw);
        const int y = (int)((id / nw) % nh);
        const int p = (int)(id / ((int64_t)nw * nh));
        const uint8_t* im = src.base + p * src.plane;
        int sy, sx;
        if (y < vp || y >= nh - vp) {            // top / bottom strips are pasted last: they win the corners
            sy = y < vp ? 0 : h - 1;
            sx = 1 + col_index[x];
        } else if (x < hp || x >= nw - hp) {
            sx = x < hp ? 0 : w - 1;
            sy = 1 + row_index[y];
        } else {
            sy = y - vp;
            sx = x - hp;
        }
        out[p * out_plane + (int64_t)y * out_pitch + x] = im[(int64_t)sy * src.pitch + sx];
    }
}

static inline int grid_of(int64_t work_items) {
    int64_t blocks = (work_items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)grid_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

}  // namespace plane
}  // namespace usdu

extern "C" {

int usdu_table_input_span(const int32_t* table, int first_out, int n_out, int* first_in, int* n_in) {
    USDU_REQUIRE(table && first_in && n_in, "usdu_table_input_span: null pointer");
    const int out_size = table[1];
    USDU_REQUIRE(first_out >= 0 && n_out > 0 && first_out + n_out <= out_size,
                 "usdu_table_input_span: outputs [%d,%d) outside the table (%d)", first_out, first_out + n_out, out_size);
    const int32_t* bounds = table + USDU_TAB_HEADER;
    int lo = bounds[2 * first_out], hi = lo;
    for (int o = first_out; o < first_out + n_out; ++o) {
        if (bounds[2 * o] < lo) lo = bounds[2 * o];
        if (bounds[2 * o] + bounds[2 * o + 1] > hi) hi = bounds[2 * o] + bounds[2 * o + 1];
    }
    *first_in = lo;
    *n_in = hi - lo;
    return USDU_OK;
}

int usdu_plane_resample_u8(const uint8_t* src, int n, int src_h, int src_w, int64_t src_pitch, int64_t src_plane,
                           const int32_t* tab_h, int ox, int ow, const int32_t* tab_v, int oy, int oh,
                           int mid_y0, int mid_rows, uint8_t* mid,
                           uint8_t* dst, int64_t dst_pitch, int64_t dst_plane, void* stream) {
    using namespace usdu;
    using namespace usdu::plane;
    USDU_REQUIRE(src && dst, "usdu_plane_resample_u8: null plane pointer");
    USDU_REQUIRE(n >= 0 && src_h > 0 && src_w > 0 && ow > 0 && oh > 0 && ox >= 0 && oy >= 0, "usdu_plane_resample_u8: bad sizes");
    USDU_REQUIRE(src_pitch >= src_w && dst_pitch >= ow, "usdu_plane_resample_u8: pitch smaller than a row");
    if (n == 0) return USDU_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const PlaneView sv{src, src_pitch, src_plane};
    if (!tab_h) USDU_REQUIRE(ox + ow <= src_w, "usdu_plane_resample_u8: window [%d,%d) outside the source width %d", ox, ox + ow, src_w);
    if (!tab_v) USDU_REQUIRE(oy + oh <= src_h, "usdu_plane_resample_u8: window [%d,%d) outside the source height %d", oy, oy + oh, src_h);
    if (!tab_h && !tab_v) {
        USDU_CUDA(launch_pdl(copy_kernel, dim3(grid_of((int64_t)n * oh * ow)), dim3(kThreads), 0, st, sv, n, oy, ox, oh, ow, dst, dst_pitch, dst_plane));
        return USDU_OK;
    }
    const int quads = (ow + 3) >> 2;
    if (!tab_v) {   // horizontal only: rows oy.. straight into dst
        USDU_CUDA(launch_pdl(hpass_kernel, dim3(grid_of((int64_t)n * oh * quads)), dim3(kThreads), 0, st, sv, n, oy, oh, tab_h, ox, ow, dst, dst_pitch, dst_plane));
        return USDU_OK;
    }
    if (!tab_h) {   // vertical only: reads the source window directly
        USDU_CUDA(launch_pdl(vpass_kernel, dim3(grid_of((int64_t)n * oh * quads)), dim3(kThreads), 0, st, sv, n, 0, ox, tab_v, oy, oh, ow, dst, dst_pitch, dst_plane));
        return USDU_OK;
    }
    USDU_REQUIRE(mid != nullptr, "usdu_plane_resample_u8: two passes need the intermediate buffer");
    USDU_REQUIRE(mid_y0 >= 0 && mid_rows > 0 && mid_y0 + mid_rows <= src_h, "usdu_plane_resample_u8: intermediate rows [%d,%d) outside the source height %d",
                 mid_y0, mid_y0 + mid_rows, src_h);
    const int64_t mid_pitch = (int64_t)quads * 4, mid_plane = mid_pitch * mid_rows;
    USDU_CUDA(launch_pdl(hpass_kernel, dim3(grid_of((int64_t)n * mid_rows * quads)), dim3(kThreads), 0, st, sv, n, mid_y0, mid_rows, tab_h, ox, ow, mid, mid_pitch, mid_plane));
    const PlaneView mv{mid, mid_pitch, mid_plane};
    USDU_CUDA(launch_pdl(vpass_kernel, dim3(grid_of((int64_t)n * oh * quads)), dim3(kThreads), 0, st, mv, n, mid_y0, 0, tab_v, oy, oh, ow, dst, dst_pitch, dst_plane));
    return USDU_OK;
}

int usdu_plane_pad_fill_u8(const uint8_t* src, int n, int h, int w, int64_t src_pitch, int64_t src_plane, int hp, int vp,
                           const int32_t* row_index, const int32_t* col_index, uint8_t* dst, int64_t dst_pitch,
                           int64_t dst_plane, void* stream) {
    using namespace usdu;
    using namespace usdu::plane;
    USDU_REQUIRE(src && dst, "usdu_plane_pad_fill_u8: null plane pointer");
    USDU_REQUIRE(n >= 0 && h > 0 && w > 0 && hp >= 0 && vp >= 0, "usdu_plane_pad_fill_u8: bad sizes");
    USDU_REQUIRE(hp == 0 || (row_index && h >= 3), "usdu_plane_pad_fill_u8: side pads need row_index and a plane of >= 3 rows");
    USDU_REQUIRE(vp == 0 || (col_index && w >= 3), "usdu_plane_pad_fill_u8: top/bottom pads need col_index and a plane of >= 3 columns");
    USDU_REQUIRE(src_pitch >= w && dst_pitch >= w + 2 * hp, "usdu_plane_pad_fill_u8: pitch smaller than a row");
    if (n == 0) return USDU_OK;
    const PlaneView sv{src, src_pitch, src_plane};
    USDU_CUDA(launch_pdl(pad_fill_kernel, dim3(grid_of((int64_t)n * (h + 2 * vp) * (w + 2 * hp))), dim3(kThreads), 0,
                         static_cast<cudaStream_t>(stream), sv, n, h, w, hp, vp, row_index, col_index, dst, dst_pitch, dst_plane));
    return USDU_OK;
}

}  // extern "C"
