// Round-to-nearest tf32 and the hi/lo split of 3xTF32, for the kernels and for the host code that builds their constant
// tables.  Plain C++ outside nvcc, so the host test (tests/test_tf32_round_host.py) compiles this very file.
//
// The tensor core TRUNCATES the low 13 mantissa bits of what it reads, which would bias every product; so both parts
// are rounded to nearest tf32 here (cvt.rna) and the hardware truncation is then a no-op: hi = rna(x), lo = rna(x - hi),
// |x - hi - lo| <= 2^-22 |x|, unbiased.  Round-to-nearest (ties away from zero, like cvt.rna.tf32.f32) is two integer
// ops on the bit pattern: add half an ulp of the 10-bit mantissa, clear the 13 low bits.  On a NaN that add can carry
// into the sign bit (0x7fffffff, the NaN arithmetic produces, becomes -0.0; 0xffffffff wraps to +0.0) or, on a payload
// held only in the low 13 bits (0x7f800001), leave Inf; so a NaN is replaced by the quiet NaN 0x7fc00000, one compare
// and one select (ptxas expands cvt.rna itself into ~5 instructions).  Inf keeps its bits, and a finite |x| at or
// above 0x7f7ff000 (within half a tf32 ulp of FLT_MAX) rounds to Inf of its sign, as cvt.rna does.
#pragma once
#include <stdint.h>
#if !defined(__CUDA_ARCH__)
#include <string.h>
#endif

#if defined(__CUDACC__)
#define FNO_TF32_HD __host__ __device__ __forceinline__
#else
#define FNO_TF32_HD inline
#endif

namespace fno {
namespace tc {

constexpr uint32_t kTf32QuietNan = 0x7fc00000u;

FNO_TF32_HD uint32_t f32_bits(float x) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(x);
#else
  uint32_t u;
  memcpy(&u, &x, 4);
  return u;
#endif
}
FNO_TF32_HD float f32_from_bits(uint32_t u) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  float x;
  memcpy(&x, &u, 4);
  return x;
#endif
}

// The bit trick alone: exact for every input that is not NaN.
FNO_TF32_HD float round_tf32_not_nan(float x) { return f32_from_bits((f32_bits(x) + 0x1000u) & 0xffffe000u); }
FNO_TF32_HD float round_tf32(float x) { return x != x ? f32_from_bits(kTf32QuietNan) : round_tf32_not_nan(x); }
// lo skips the NaN test: when x - hi is NaN, hi is already NaN or Inf, so hi * b + lo * b is non-finite whatever lo is.
FNO_TF32_HD void split_tf32(float x, float& hi, float& lo) {
  hi = round_tf32(x);
  lo = round_tf32_not_nan(x - hi);
}

}  // namespace tc
}  // namespace fno
