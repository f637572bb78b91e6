// usdu_tma.cuh -- Tensor Memory Accelerator plumbing (sm_90a): 2-D tiled tensor maps over the
// u8 canvas, bulk-tensor loads into shared memory signalled through an mbarrier, bulk-tensor
// stores back.  Inline PTX only (no CUTLASS); the host encoder is resolved through
// cudaGetDriverEntryPoint so the library does not link libcuda.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace usdu {
namespace tma {

// ---- host ---------------------------------------------------------------------------------
// Tensor map of a u8 image stack: inner dimension = `row_bytes` bytes, outer = `rows`, row pitch
// `pitch` bytes (multiple of 16), box = box_bytes x box_rows.  Returns false on failure.
inline bool encode_u8_2d(CUtensorMap* map, const void* base, uint64_t row_bytes, uint64_t rows, uint64_t pitch,
                         uint32_t box_bytes, uint32_t box_rows) {
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return false;
        fn = reinterpret_cast<EncodeFn>(p);
    }
    const cuuint64_t dims[2] = {row_bytes, rows};
    const cuuint64_t strides[1] = {pitch};
    const cuuint32_t box[2] = {box_bytes, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Same image stack as a 3-D tensor {row_bytes, rows_per_frame, frames}: boxes are clipped at the
// bottom of their own frame (a 2-D {row_bytes, frames*rows} view would let a block at the bottom of
// frame b read -- and, on store, overwrite -- the top rows of frame b+1).  Box = box_bytes x box_rows x 1.
inline bool encode_u8_3d(CUtensorMap* map, const void* base, uint64_t row_bytes, uint64_t rows, uint64_t frames,
                         uint64_t pitch, uint32_t box_bytes, uint32_t box_rows) {
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return false;
        fn = reinterpret_cast<EncodeFn>(p);
    }
    const cuuint64_t dims[3] = {row_bytes, rows, frames};
    const cuuint64_t strides[2] = {pitch, pitch * rows};
    const cuuint32_t box[3] = {box_bytes, box_rows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// ---- device -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// global (tensor map, coordinates x = byte column, y = row) -> shared, completes on `bar`
__device__ __forceinline__ void load_2d(void* smem_dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(bar)) : "memory");
}

// shared -> global through the tensor map; call fence_async_smem() after the last generic write
__device__ __forceinline__ void store_2d(const CUtensorMap* map, int x, int y, const void* smem_src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(smem_src)) : "memory");
}

__device__ __forceinline__ void load_3d(void* smem_dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void store_3d(const CUtensorMap* map, int x, int y, int z, const void* smem_src) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%1, %2, %3}], [%4];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(z), "r"(smem_u32(smem_src)) : "memory");
}

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// enough before a CTA exits: the bulk store has finished READING shared memory (the global writes
// complete by the end of the grid like any other store)
__device__ __forceinline__ void store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

}  // namespace tma
}  // namespace usdu
