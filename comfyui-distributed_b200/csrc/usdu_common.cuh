// usdu_common.cuh -- shared declarations for libusdu_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/usdu_b200.h"

namespace usdu {

constexpr int kPrecisionBits = 32 - 8 - 2;  // Pillow Resample.c PRECISION_BITS
constexpr int BW = USDU_BLOCK_W;            // canvas / output block, pixels
constexpr int BH = USDU_BLOCK_H;
constexpr int kThreads = 256;

void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
// SMs of the current device (cudaDevAttrMultiProcessorCount, cached per device), or a negative usdu_status.
int sm_count();
// the same for sizing grids: at least 1 (a failed query leaves the error to the launch that follows)
inline int grid_sms() { const int n = sm_count(); return n > 0 ? n : 1; }

#define USDU_REQUIRE(cond, ...)                      \
    do {                                             \
        if (!(cond)) {                               \
            ::usdu::set_error(__VA_ARGS__);          \
            return USDU_ERR_INVALID;                 \
        }                                            \
    } while (0)

#define USDU_CUDA(call)                                              \
    do {                                                             \
        int _s = ::usdu::check_cuda((call), #call);                  \
        if (_s != USDU_OK) return _s;                                \
    } while (0)

// Let kernel `fn` launch with `bytes` of dynamic shared memory on the current device: raise its limit, never lower it.
// A launch captured into a CUDA graph keeps its size after later, smaller launches of the same kernel; a limit lowered
// below it makes the runtime reject that node (cudaGraphKernelNodeSetAttribute, instantiation: "invalid argument").
inline int raise_smem_limit(const void* fn, size_t bytes) {
    if (bytes <= 48 * 1024) return USDU_OK;
    cudaFuncAttributes a;
    USDU_CUDA(cudaFuncGetAttributes(&a, fn));
    if ((size_t)a.maxDynamicSharedSizeBytes < bytes)
        USDU_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return USDU_OK;
}

// (uint8)(255.f * x): fp32 multiply (round to nearest), C truncation, wrap to 8 bits.
// utils/image.py:8-10 -- numpy's float32 -> uint8 cast on x86: cvttss2si, then the low byte.  cvttss2si returns
// 0x80000000 for NaN, +-inf and every product outside [-2^31, 2^31), so all of those give 0.  cvt.rzi.s32 gives 0
// for NaN and 0x80000000 below the range, but saturates to 0x7FFFFFFF above it (255 for the low byte), so products
// >= 2^31 (and +inf) are replaced by 0 before the conversion: one FSETP + FSEL, and the bytes are still packed with
// PRMT (a compare on the integer result costs more and made blend_fast_kernel spill).  Checked against numpy's rule
// for all 2^32 fp32 inputs in tests/test_gpu_casts.py.
__device__ __forceinline__ uint32_t quant_u8(float x) {
    const float p = __fmul_rn(255.0f, x);
    return static_cast<uint32_t>(__float2int_rz(p < 2147483648.0f ? p : 0.0f)) & 0xFFu;
}

// u / 255.0f with IEEE division (utils/image.py:13).
__device__ __forceinline__ float dequant_u8(uint32_t u) {
    return __fdiv_rn(static_cast<float>(u), 255.0f);
}

// The same value without a divide, a conversion or a table: the byte goes into the mantissa
// of 2^23 (one LOP), one FADD removes the bias, then q0 = x*rcp, r = fma(-255, q0, x) (exact),
// q = fma(r, rcp, q0) is the correctly rounded quotient (Markstein); checked for all 256
// codes against __fdiv_rn in tests/test_gpu_parity.py::test_quantize_dequantize.
__device__ __forceinline__ float dequant_u8_fast(uint32_t u) {
    const float x = __uint_as_float(0x4B000000u | u) - 8388608.0f;
    const float rcp = 0.003921568859368563f;   // fp32(1/255)
    const float q0 = __fmul_rn(x, rcp);
    const float r = __fmaf_rn(-255.0f, q0, x);
    return __fmaf_rn(r, rcp, q0);
}

// Store of an fp32 tile hand-off (the crop's output): the sampler, the next kernel on the stream, reads it right away, so
// it is stored with an L2 evict_last policy instead of the evict-first hint of a streaming result.  On cfg2 it beats
// both the evict-first and a plain store (measured on an H100 80GB HBM3 at 400 W, DESIGN section 9.1).
__device__ __forceinline__ void store_handoff(float* p, float4 v) {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w),
                 "l"(pol) : "memory");
}

__device__ __forceinline__ uint32_t clip8(int v) {
    return static_cast<uint32_t>(min(max(v, 0), 255));
}

// AlphaComposite.c with an opaque destination (see oracle/usdu_oracle.py composite_u8).
__device__ __forceinline__ uint32_t composite8(uint32_t S, uint32_t D, uint32_t A) {
    uint32_t tmp = S * (A * 128u) + D * ((255u - A) * 128u) + (0x80u << 7);
    tmp = ((tmp >> 8) + tmp) >> 8;
    return tmp >> 7;
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------
// Every kernel of the wave loop reads only STATIC data (job records, tables) in its prologue.
// pdl_launch_dependents() lets the next kernel of the stream start being scheduled while this
// one is still running; pdl_wait() (griddepcontrol.wait) blocks until the previous kernel has
// completed and flushed, and must precede the first access to data that kernel produced.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Launch with the programmatic-stream-serialization attribute (captured as a programmatic edge
// inside CUDA graphs).  USDU_NO_PDL=1 in the environment falls back to plain launches.
template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    static int use = -1;
    if (use < 0) { const char* e = getenv("USDU_NO_PDL"); use = (e && e[0] == '1') ? 0 : 1; }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = use ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

struct TableView {
    int in_size, out_size, ksize;
    const int32_t* bounds;  // out_size x 2
    const int32_t* kk;      // out_size x ksize
};

__device__ __forceinline__ TableView table_at(const int32_t* tabs, int off) {
    TableView t;
    const int32_t* p = tabs + off;
    t.in_size = p[0];
    t.out_size = p[1];
    t.ksize = p[2];
    t.bounds = p + USDU_TAB_HEADER;
    t.kk = t.bounds + 2 * t.out_size;
    return t;
}

}  // namespace usdu
