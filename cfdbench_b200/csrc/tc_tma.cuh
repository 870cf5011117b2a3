// 2-D TMA tensor loads (cp.async.bulk.tensor, completion on an mbarrier) and the encoding of their tensor maps, shared
// by the TMA-fed kernels (fno_mode_mix.cu, fno_dft_fwd_tc.cu).
#pragma once
#include "fno_common.cuh"
#include <cuda.h>

namespace fno {

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                   smem_u32(dst)),
               "l"(tm), "r"(c0), "r"(c1), "r"(smem_u32(bar))
               : "memory");
}

// Row-major 2-D tensor [rows][inner] (row pitch = inner elements), box {box_inner, box_rows}, 128-byte swizzle: every
// box row is one 128-byte line, and the 16-byte chunk c of line r lands at chunk position c ^ (r & 7).
typedef CUresult (*TmaEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline cudaError_t make_tma_map_2d(CUtensorMap* out, CUtensorMapDataType dtype, size_t elt_bytes, const void* base,
                                   uint64_t inner, uint64_t rows, uint32_t box_inner, uint32_t box_rows) {
  static TmaEncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess) return e;
    if (!p) return cudaErrorNotSupported;
    fn = reinterpret_cast<TmaEncodeFn>(p);
  }
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(inner * elt_bytes)};
  const cuuint32_t box[2] = {box_inner, box_rows}, estr[2] = {1, 1};
  const CUresult r = fn(out, dtype, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

}  // namespace fno
