// Shared definitions for the sm_90a FNO kernels (cfdbench_b200).
//
// Problem constants are the reference's FNO configuration (reference src/args.py:99-103,187-197:
// 64x64 grid, fno_hidden_dim=32, fno_modes_x=fno_modes_y=12).  Other grids run the runtime-(H, W) kernels of
// fno_grid.cu; the Python wrapper rejects anything else, there is no CPU fallback.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace fno {

constexpr int kH = 64;
constexpr int kW = 64;
constexpr int kHW = kH * kW;
constexpr int kC = 32;        // hidden channels
constexpr int kM1 = 12;       // kept |kx| modes per corner
constexpr int kM2 = 12;       // kept ky modes
constexpr int kKX = 2 * kM1;  // kept kx rows: 0..11 (weights1) and 52..63 (weights2)
constexpr int kModes = kKX * kM2;  // 288 complex modes per (sample, channel)
constexpr int kProj = 128;    // fc1 width (reference fno2d.py:175)
constexpr int kMaxCaseParams = 16;

// ------------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk-copy (TMA engine, SASS UBLKCP) wrappers.  A plane of an NCHW activation is a
// contiguous 16 KB (fp32) / 8 KB (bf16) run, so plain bulk copies are enough: no tensor map needed.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {  // release.cta: prior writes of this thread are visible
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a wrong transaction count / descriptor must surface as a CUDA error (trap), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 22)) __trap();
  }
}

// ------------------------------------------------------------------------------------------------
// Programmatic dependent launch.  The six kernels of a rollout step form one dependency chain on one
// stream; each is launched with cudaLaunchAttributeProgrammaticStreamSerialization so that its CTAs
// may become resident -- and run their prologue: barrier init, constant tables, weight staging --
// while the previous kernel drains.  Rules every chained kernel follows:
//   * pdl_wait() (griddepcontrol.wait: the previous grid has completed and its writes are visible)
//     comes before the first access to anything a kernel of the chain writes, and every CTA executes it;
//   * pdl_launch_dependents() is issued only AFTER pdl_wait(), so at most two kernels overlap and the
//     next kernel's prologue may read anything written two or more launches earlier (packed weights);
//   * the prologue before pdl_wait() reads only weights / constant tables and writes only shared memory.
// Without the launch attribute both instructions are no-ops, so the same kernels serve the training path.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <bool kEarly = true, typename... KArgs, typename... Args>
inline cudaError_t launch_chained(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                  Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = kEarly ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ------------------------------------------------------------------------------------------------
// Per-DEVICE launcher state (one process may drive several GPUs): the opt-in dynamic shared-memory size is a per-device
// function attribute and the SM count differs per device, so both are cached per device index, not per process.
// ------------------------------------------------------------------------------------------------
struct PerDeviceLaunch {
  bool done[64] = {};
  int n_sm[64] = {};
};
template <typename Kern>
inline cudaError_t per_device_setup(Kern kern, size_t smem, PerDeviceLaunch& st, int* n_sm = nullptr) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!st.done[dev]) {
    if (smem > 0) {
      e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
      if (e != cudaSuccess) return e;
    }
    e = cudaDeviceGetAttribute(&st.n_sm[dev], cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    st.done[dev] = true;
  }
  if (n_sm) *n_sm = st.n_sm[dev];
  return cudaSuccess;
}

// ------------------------------------------------------------------------------------------------
// Activation storage types.  Arithmetic is always fp32; TAct only selects how hidden activations
// are stored in HBM between kernels (float = parity mode, bf16 = BASELINE.json's bf16 batches).
// ------------------------------------------------------------------------------------------------
template <typename T>
struct Act;
template <>
struct Act<float> {
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <>
struct Act<__nv_bfloat16> {
  static __device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
};

// Fused multiply-add on a pair of floats: two correctly rounded FFMA, so the pair form of the GELU / fc2 code gives
// the same bits as the scalar form.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// ------------------------------------------------------------------------------------------------
// Exact (erf) GELU, nn.GELU() default (reference fno2d.py:147), evaluated without erff():
//   GELU(x) = max(x,0) - 0.5|x| * erfc(|x|/sqrt2),   erfc(z) = 2^{p(z)}, p = degree-8 minimax fit
// |exp2(p)-erfc| <= 1.5e-8 on [0,4.5]; beyond that erfc < 2e-10 and p keeps decreasing (no clamp needed).  In fp32 the result
// is within 2.7e-7 abs of the float64 GELU (torch's own fp32 GELU: 1.3e-6), see tests/test_gelu.py.
// One MUFU.EX2 + 8 FFMA per element, branch-free.
// ------------------------------------------------------------------------------------------------
#define FNO_GELU_C0 2.1715042208825253e-08f
#define FNO_GELU_C1 -1.6279093256885822f
#define FNO_GELU_C2 -0.918409818247829f
#define FNO_GELU_C3 -0.1485066268693784f
#define FNO_GELU_C4 0.028301834411822168f
#define FNO_GELU_C5 -0.0008250955854016083f
#define FNO_GELU_C6 -0.001460431044966736f
#define FNO_GELU_C7 0.0004369618322752869f
#define FNO_GELU_C8 -4.4355305747040687e-05f

__device__ __forceinline__ float ex2_approx(float x) {  // 2^x, one MUFU.EX2 (x <= 0 here: no overflow, ftz is fine)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// p(z) ~ log2(erfc(z)); its leading coefficient is negative and p is monotone beyond the fit range, so no clamp
// is needed: 2^p just underflows to 0 for large z.
__device__ __forceinline__ float erfc_poly(float z) {
  float p = FNO_GELU_C8;
  p = fmaf(p, z, FNO_GELU_C7);
  p = fmaf(p, z, FNO_GELU_C6);
  p = fmaf(p, z, FNO_GELU_C5);
  p = fmaf(p, z, FNO_GELU_C4);
  p = fmaf(p, z, FNO_GELU_C3);
  p = fmaf(p, z, FNO_GELU_C2);
  p = fmaf(p, z, FNO_GELU_C1);
  p = fmaf(p, z, FNO_GELU_C0);
  return p;
}
__device__ __forceinline__ float erfc_abs_scaled(float ax) {  // erfc(ax/sqrt2), ax >= 0
  return ex2_approx(erfc_poly(ax * 0.70710678118654752f));
}
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  return fmaf(z * -0.70710678118654752f, ex2_approx(erfc_poly(z)), fmaxf(x, 0.f));
}
// d/dx GELU(x) = Phi(x) + x phi(x)
__device__ __forceinline__ float dgelu_erf(float x) {
  const float ax = fabsf(x);
  const float e = 0.5f * erfc_abs_scaled(ax);
  const float cdf = x >= 0.f ? 1.f - e : e;
  const float pdf = 0.3989422804014327f * ex2_approx(-0.7213475204444817f * x * x);
  return fmaf(x, pdf, cdf);
}

// Pair version.  The same polynomial re-expressed in a = |x| with the 1/2 folded into the
// exponent:  q(a) = p(a / sqrt2) - 1,  D_k = C_k 2^{-k/2} (D_0 = C_0 - 1),  so  2^{q(|x|)} = erfc(|x|/sqrt2) / 2  and
//   GELU(x) = max(x,0) - |x| 2^{q(|x|)}.
// Per pair: 9 fma pairs (the version in z = |x|/sqrt2 needs 12), 2 MUFU, and |x| / max(x,0).  Accuracy is unchanged
// (2.7e-7 max abs, tests/test_host.py).
#define FNO_GELU_D0 -0.9999999782849578f
#define FNO_GELU_D1 -1.1511057233512165f
#define FNO_GELU_D2 -0.4592049091239145f
#define FNO_GELU_D3 -0.05250502145523891f
#define FNO_GELU_D4 0.007075458602955542f
#define FNO_GELU_D5 -0.00014585767089114035f
#define FNO_GELU_D6 -0.000182553880620842f
#define FNO_GELU_D7 3.8622334340194274e-05f
#define FNO_GELU_D8 -2.772206609190043e-06f
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
  const float2 a = make_float2(fabsf(x.x), fabsf(x.y));
  float2 p = make_float2(FNO_GELU_D8, FNO_GELU_D8);
  p = ffma2(p, a, make_float2(FNO_GELU_D7, FNO_GELU_D7));
  p = ffma2(p, a, make_float2(FNO_GELU_D6, FNO_GELU_D6));
  p = ffma2(p, a, make_float2(FNO_GELU_D5, FNO_GELU_D5));
  p = ffma2(p, a, make_float2(FNO_GELU_D4, FNO_GELU_D4));
  p = ffma2(p, a, make_float2(FNO_GELU_D3, FNO_GELU_D3));
  p = ffma2(p, a, make_float2(FNO_GELU_D2, FNO_GELU_D2));
  p = ffma2(p, a, make_float2(FNO_GELU_D1, FNO_GELU_D1));
  p = ffma2(p, a, make_float2(FNO_GELU_D0, FNO_GELU_D0));
  const float2 h = make_float2(ex2_approx(p.x), ex2_approx(p.y));  // erfc(|x|/sqrt2) / 2
  return ffma2(make_float2(-a.x, -a.y), h, make_float2(fmaxf(x.x, 0.f), fmaxf(x.y, 0.f)));
}

// Degree-5 variant of the pair GELU for the project kernel in bf16 storage mode (project_tc_kernel<bf16>), whose epilogue
// -- 134 M GELUs per launch at B=256 -- is bound by the fma pipe; three fewer fma per element.
// q(a) ~ log2(erfc(a/sqrt2)/2), weighted minimax fit of the GELU error on [0, 8], negative leading coefficient (2^q underflows
// beyond the fit range, no clamp).  fp32 result within 6.4e-7 abs of the float64 GELU -- torch's own fp32 nn.GELU() is at
// 1.3e-6 -- checked by tests/test_host.py.  Used ONLY where the output is not fed back through further layers in fp32
// parity mode: with it everywhere the fp32-storage rel-L2 against the reference rose from 2.2e-7 to 2.1e-6 (measured), so
// the Fourier blocks and the fp32-storage project keep the degree-8 fit above.
#define FNO_GELU_E0 -1.0000376366992503f
#define FNO_GELU_E1 -1.1507877474081256f
#define FNO_GELU_E2 -0.45999268192636272f
#define FNO_GELU_E3 -0.051827144796875543f
#define FNO_GELU_E4 0.0070844550401877602f
#define FNO_GELU_E5 -0.00047329356073930895f
// N pairs at once, coefficient loop outside (N independent Horner chains)
template <int N>
__device__ __forceinline__ void gelu_erf2_deg5_batch(float2 (&x)[N]) {
  float2 p[N];
  constexpr float kE[6] = {FNO_GELU_E0, FNO_GELU_E1, FNO_GELU_E2, FNO_GELU_E3, FNO_GELU_E4, FNO_GELU_E5};
#pragma unroll
  for (int i = 0; i < N; ++i)
    p[i] = ffma2(make_float2(kE[5], kE[5]), make_float2(fabsf(x[i].x), fabsf(x[i].y)), make_float2(kE[4], kE[4]));
#pragma unroll
  for (int k = 3; k >= 0; --k)
#pragma unroll
    for (int i = 0; i < N; ++i)
      p[i] = ffma2(p[i], make_float2(fabsf(x[i].x), fabsf(x[i].y)), make_float2(kE[k], kE[k]));
#pragma unroll
  for (int i = 0; i < N; ++i) p[i] = make_float2(ex2_approx(p[i].x), ex2_approx(p[i].y));   // erfc(|x|/sqrt2) / 2
#pragma unroll
  for (int i = 0; i < N; ++i)
    x[i] = ffma2(make_float2(-fabsf(x[i].x), -fabsf(x[i].y)), p[i], make_float2(fmaxf(x[i].x, 0.f), fmaxf(x[i].y, 0.f)));
}

// status codes of the C ABI
enum : int { kOk = 0, kErrArg = 1, kErrCuda = 2, kErrUnsupported = 3 };

}  // namespace fno
