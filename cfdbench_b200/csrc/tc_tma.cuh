// TMA tensor loads (cp.async.bulk.tensor, completion on an mbarrier), TMA tensor stores (bulk groups) and the encoding of
// their tensor maps, shared by the TMA-fed kernels (fno_mode_mix.cu, fno_dft_fwd_tc.cu, fno_block_fused.cu).
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
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          smem_u32(dst)),
      "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
// Store of one box from shared memory.  The writing threads make their shared-memory stores visible to the async proxy
// (fence.proxy.async.shared::cta) and synchronise before one thread issues it; stores are tracked as bulk groups.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tm),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most kPending of this thread's bulk groups still read shared memory
template <int kPending>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kPending) : "memory");
}
// at most kPending of this thread's bulk groups are incomplete (their global writes included)
template <int kPending>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(kPending) : "memory");
}

typedef CUresult (*TmaEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline cudaError_t tma_encode_fn(TmaEncodeFn* out) {
  static TmaEncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess) return e;
    if (!p) return cudaErrorNotSupported;
    fn = reinterpret_cast<TmaEncodeFn>(p);
  }
  *out = fn;
  return cudaSuccess;
}

// Row-major 2-D tensor [rows][inner] (row pitch = inner elements), box {box_inner, box_rows}, 128-byte swizzle: every
// box row is one 128-byte line, and the 16-byte chunk c of line r lands at chunk position c ^ (r & 7).
inline cudaError_t make_tma_map_2d(CUtensorMap* out, CUtensorMapDataType dtype, size_t elt_bytes, const void* base,
                                   uint64_t inner, uint64_t rows, uint32_t box_inner, uint32_t box_rows) {
  TmaEncodeFn fn = nullptr;
  cudaError_t e = tma_encode_fn(&fn);
  if (e != cudaSuccess) return e;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(inner * elt_bytes)};
  const cuuint32_t box[2] = {box_inner, box_rows}, estr[2] = {1, 1};
  const CUresult r = fn(out, dtype, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// Dense 3-D tensor [d2][d1][d0] (d0 contiguous), box {box0, box1, box2}, 128-byte swizzle: box0 * elt_bytes must be at
// most 128, every (d1, d2) line of the box is one line of the shared-memory image, swizzled as above.
inline cudaError_t make_tma_map_3d(CUtensorMap* out, CUtensorMapDataType dtype, size_t elt_bytes, const void* base,
                                   uint64_t d0, uint64_t d1, uint64_t d2, uint32_t box0, uint32_t box1, uint32_t box2) {
  TmaEncodeFn fn = nullptr;
  cudaError_t e = tma_encode_fn(&fn);
  if (e != cudaSuccess) return e;
  const cuuint64_t gdim[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1), static_cast<cuuint64_t>(d2)};
  const cuuint64_t gstride[2] = {static_cast<cuuint64_t>(d0 * elt_bytes), static_cast<cuuint64_t>(d0 * d1 * elt_bytes)};
  const cuuint32_t box[3] = {box0, box1, box2}, estr[3] = {1, 1, 1};
  const CUresult r = fn(out, dtype, 3, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

}  // namespace fno
