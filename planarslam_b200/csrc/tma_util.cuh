// TMA (cp.async.bulk.tensor) + mbarrier helpers for sm_90a, and the host-side tensor-map encoder.
//
// Image / depth tiles are staged into shared memory by the tensor memory accelerator: one elected thread arms an mbarrier with the
// byte count of the box and issues the bulk tensor copy; the copy engine zero-fills whatever part of the box lies outside the tensor
// (the kernels then rebuild OpenCV's REFLECT_101 border from the interior that is already in the tile), and the CTA waits on the
// barrier's phase.  No thread issues per-byte global loads.  The driver entry point cuTensorMapEncodeTiled is resolved through
// cudaGetDriverEntryPoint, so the library has no link-time dependency on libcuda.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace pslam {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");       // make the initialised barrier visible to the async proxy
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// box of a rank-3 tensor (x, y, frame) -> shared memory; completion is signalled on `bar` (complete_tx of the box bytes)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(smem_dst)),
                 "l"(map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
                 : "memory");
}

// Host: rank-3 tiled tensor map over `n` images of w x h elements of `elem_bytes` bytes (row pitch and image stride in bytes, both
// multiples of 16; base 16-byte aligned).  Out-of-bounds box elements are filled with zeros.  Returns false when the driver refuses.
inline bool tma_encode_3d(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes, const void* base, int w, int h, int n, size_t pitch_bytes,
                          size_t image_stride_bytes, int box_w, int box_h) {
    typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static encode_fn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
        return (encode_fn)p;
    }();
    if (!fn || ((uintptr_t)base & 15) || (pitch_bytes & 15) || (image_stride_bytes & 15) || ((size_t)box_w * elem_bytes & 15) || box_w > 256 || box_h > 256) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
    const cuuint64_t strides[2] = {(cuuint64_t)pitch_bytes, (cuuint64_t)image_stride_bytes};
    const cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(out, dtype, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace pslam
