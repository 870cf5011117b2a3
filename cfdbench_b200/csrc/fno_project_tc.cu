// Project kernel on the tensor cores: preds = (fc2 . GELU . fc1)(a_L) * mask
// replacing Conv2d(32,128,1) + GELU + Conv2d(128,2,1) + "* mask" (reference src/models/fno/fno2d.py:228-233).
//
// fc1 is the one genuinely dense GEMM of the model (16.8 MFMA per sample): per tile of 64 pixels (one image row)
//     D[64 px][128 hidden] = A[64 px][32 ch] * W1^T         (wgmma m64n128k8 tf32, K = 32)
// run as 3xTF32 (hi*hi + lo*hi + hi*lo, round-to-nearest split) so the result stays within 1e-6 of fp32; bf16 activations
// are exact in tf32, so that storage mode needs two passes (x*W1_hi + x*W1_lo).  The (B,128,64,64) hidden tensor of the
// reference (537 MB at B=256) exists only in the accumulator registers: the epilogue adds b1, applies the GELU (degree-8
// erfc fit; the degree-5 fit in bf16 storage mode, fno_common.cuh), contracts with fc2 and sums the partial sums of the
// four lanes that share a pixel in a fixed order (deterministic results).
//
// Persistent CTA of four independent warpgroup pipelines.  Per tile: the activation values prefetched into registers one
// tile ahead (coalesced loads) are split into tf32 hi/lo and written as the K-major A operand; the warpgroup issues the
// MMAs, waits for them and runs the epilogue while the other pipelines of the SM load, multiply or compute their GELUs.
#include "fno_common.cuh"
#include "tc_common.cuh"

namespace fno {

constexpr int kPtWG = 4;
constexpr int kPtThreads = 128 * kPtWG;
constexpr int kPtM = kW;                                   // pixels per tile (one image row)
constexpr uint32_t kPtLboA = (kPtM / 8) * 128;             // 1024
constexpr uint32_t kPtLboB = (kProj / 8) * 128;            // 2048 (B operand has 128 rows = hidden units)
constexpr int kPtTilesPerSample = kH;                      // 64
constexpr int kPtReps = kPtM * (kC / 4) / 128;             // 4 activation tasks per thread

struct PtSmem {
  alignas(128) float w_hi[kProj * kC];       // 16 KB   B operand: [n = hidden j][k = channel i]
  alignas(128) float w_lo[kProj * kC];       // 16 KB
  alignas(128) float a_hi[kPtWG][kPtM * kC]; // 4 x 8 KB
  alignas(128) float a_lo[kPtWG][kPtM * kC]; // 4 x 8 KB
  alignas(16) float4 w2q[kProj / 2];         // (w2[0][j], w2[1][j], w2[0][j+1], w2[1][j+1])
  alignas(16) float2 b1p[kProj / 2];         // (b1[j], b1[j+1])
};

// Activation values of one tile held by a thread between the prefetch and the split pass.
// task = rep*128 + t -> (pixel m = task & 63, channel quad kq = task >> 6): lanes run over consecutive pixels,
// so the global loads coalesce and the 16-byte operand stores are conflict-free.
template <typename TAct>
struct PtRegs {
  TAct v[kPtReps][4];
};

template <typename TAct>
__device__ __forceinline__ void pt_prefetch(PtRegs<TAct>& r, const TAct* __restrict__ a, int tile, int t) {
  const int b = tile / kPtTilesPerSample, p0 = (tile % kPtTilesPerSample) * kPtM;
#pragma unroll
  for (int rep = 0; rep < kPtReps; ++rep) {
    const int task = rep * 128 + t;
    const int m = task & (kPtM - 1), kq = task >> 6;
    const TAct* src = a + (static_cast<size_t>(b) * kC + 4 * kq) * kHW + p0 + m;
#pragma unroll
    for (int c = 0; c < 4; ++c) r.v[rep][c] = __ldg(src + static_cast<size_t>(c) * kHW);
  }
}

__device__ __forceinline__ float pt_to_float(float v) { return v; }
__device__ __forceinline__ float pt_to_float(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename TAct>
__device__ __forceinline__ void pt_split_store(const PtRegs<TAct>& r, float* a_hi, float* a_lo, int t) {
#pragma unroll
  for (int rep = 0; rep < kPtReps; ++rep) {
    const int task = rep * 128 + t;
    const int m = task & (kPtM - 1), kq = task >> 6;
    float hi[4], lo[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float x = pt_to_float(r.v[rep][c]);
      if constexpr (sizeof(TAct) == 4) tc::split_tf32(x, hi[c], lo[c]);
      else hi[c] = x;  // bf16 is tf32-exact: no lo part
    }
    const uint32_t off = tc::kmajor_offset(m, 4 * kq, kPtM) / 4;
    *reinterpret_cast<float4*>(a_hi + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
    if constexpr (sizeof(TAct) == 4) *reinterpret_cast<float4*>(a_lo + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
  }
}

template <typename TAct>
__global__ void __launch_bounds__(kPtThreads, 1)
    project_tc_kernel(const TAct* __restrict__ a, const float* __restrict__ w1, const float* __restrict__ b1,
                      const float* __restrict__ w2, const float* __restrict__ b2, const float* __restrict__ mask,
                      float* __restrict__ preds, int n_tiles) {
  constexpr bool kBf16 = sizeof(TAct) == 2;
  extern __shared__ __align__(1024) unsigned char smem_raw[];  // no pointer arithmetic: keeps LDS/STS addressing
  PtSmem& sm = *reinterpret_cast<PtSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tc::warp_index_uniform() >> 2, t = tid & 127, wq = (tid >> 5) & 3;

  for (int e = tid; e < kProj * kC; e += kPtThreads) {  // w1[j][i] -> B[n = j][k = i]
    const int j = e / kC, i = e % kC;
    float hi, lo;
    tc::split_tf32(w1[e], hi, lo);
    const uint32_t off = tc::kmajor_offset(j, i, kProj) / 4;
    sm.w_hi[off] = hi;
    sm.w_lo[off] = lo;
  }
  if (tid < kProj / 2) {
    sm.w2q[tid] = make_float4(w2[2 * tid], w2[kProj + 2 * tid], w2[2 * tid + 1], w2[kProj + 2 * tid + 1]);
    sm.b1p[tid] = make_float2(b1[2 * tid], b1[2 * tid + 1]);
  }
  const float b2x = b2[0], b2y = b2[1];
  tc::fence_proxy_async_smem();   // the constant operands above are read by the tensor cores
  __syncthreads();
  pdl_wait();  // fc1 / fc2 weights above are not produced by the chain; the activations are
  pdl_launch_dependents();

  const int first = blockIdx.x * kPtWG + wg, stride = gridDim.x * kPtWG;
  float* a_hi = sm.a_hi[wg];
  float* a_lo = sm.a_lo[wg];
  PtRegs<TAct> regs;
  if (first < n_tiles) pt_prefetch<TAct>(regs, a, first, t);
  for (int tile = first; tile < n_tiles; tile += stride) {
    // the A operand was last read by this pipeline's previous MMAs, which every thread waited for
    pt_split_store<TAct>(regs, a_hi, a_lo, t);
    tc::fence_proxy_async_smem();
    tc::named_barrier(1 + wg, 128);
    // prefetch AFTER the fence: the membar inside fence.proxy.async would otherwise wait for these loads
    if (tile + stride < n_tiles) pt_prefetch<TAct>(regs, a, tile + stride, t);
    float acc[64];
    tc::wg_fence();
    {
      const uint32_t a_s[3] = {tc::smem_addr(a_hi), tc::smem_addr(a_lo), tc::smem_addr(a_hi)};
      const uint32_t b_s[3] = {tc::smem_addr(sm.w_hi), tc::smem_addr(sm.w_hi), tc::smem_addr(sm.w_lo)};
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {
        if (kBf16 && pass == 1) continue;
#pragma unroll
        for (int ks = 0; ks < kC / 8; ++ks)
          tc::wg_tf32_ss_n128(acc, tc::make_smem_desc(a_s[pass] + ks * 2 * kPtLboA, kPtLboA, 128),
                              tc::make_smem_desc(b_s[pass] + ks * 2 * kPtLboB, kPtLboB, 128), (pass | ks) ? 1u : 0u);
      }
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc);
    // epilogue: acc[4 i + 2 hh + e] = D[px = 16 wq + lane/4 + 8 hh][j = 8 i + 2 (lane%4) + e]
    const int b = tile / kPtTilesPerSample, p0 = (tile % kPtTilesPerSample) * kPtM;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float2 out = make_float2(0.f, 0.f);   // (out channel 0, out channel 1)
#pragma unroll
      for (int i0 = 0; i0 < 16; i0 += 8) {  // 8 pairs at a time: 8 independent polynomial chains in flight
        float2 g[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float2 bb = sm.b1p[4 * (i0 + i) + (lane & 3)];
          g[i] = make_float2(acc[4 * (i0 + i) + 2 * hh] + bb.x, acc[4 * (i0 + i) + 2 * hh + 1] + bb.y);
        }
        if constexpr (kBf16) {
          gelu_erf2_deg5_batch<8>(g);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) g[i] = gelu_erf2(g[i]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 wq4 = sm.w2q[4 * (i0 + i) + (lane & 3)];
          out = ffma2(make_float2(g[i].x, g[i].x), make_float2(wq4.x, wq4.y), out);
          out = ffma2(make_float2(g[i].y, g[i].y), make_float2(wq4.z, wq4.w), out);
        }
      }
      // the four lanes of a pixel hold disjoint hidden units: fixed-order butterfly sum
      out.x += __shfl_xor_sync(0xffffffffu, out.x, 1);
      out.y += __shfl_xor_sync(0xffffffffu, out.y, 1);
      out.x += __shfl_xor_sync(0xffffffffu, out.x, 2);
      out.y += __shfl_xor_sync(0xffffffffu, out.y, 2);
      if ((lane & 3) == 0) {
        const int pix = p0 + 16 * wq + (lane >> 2) + 8 * hh;
        const float mk = __ldg(mask + static_cast<size_t>(b) * kHW + pix);
        preds[(static_cast<size_t>(b) * 2 + 0) * kHW + pix] = (b2x + out.x) * mk;
        preds[(static_cast<size_t>(b) * 2 + 1) * kHW + pix] = (b2y + out.y) * mk;
      }
    }
  }
}

template <typename TAct>
cudaError_t launch_project_tc(const void* a, const float* w1, const float* b1, const float* w2, const float* b2,
                              const float* mask, float* preds, int batch, cudaStream_t stream) {
  auto kern = project_tc_kernel<TAct>;
  constexpr size_t smem = sizeof(PtSmem);
  static PerDeviceLaunch pd;
  int n_sm = 0;
  cudaError_t e0 = per_device_setup(kern, smem, pd, &n_sm);
  if (e0 != cudaSuccess) return e0;
  const int n_tiles = batch * kPtTilesPerSample;
  const int want = (n_tiles + kPtWG - 1) / kPtWG;
  const int grid = want < n_sm ? want : n_sm;
  return launch_chained(kern, dim3(grid), dim3(kPtThreads), smem, stream, static_cast<const TAct*>(a), w1, b1, w2, b2,
                        mask, preds, n_tiles);
}
template cudaError_t launch_project_tc<float>(const void*, const float*, const float*, const float*, const float*,
                                              const float*, float*, int, cudaStream_t);
template cudaError_t launch_project_tc<__nv_bfloat16>(const void*, const float*, const float*, const float*,
                                                      const float*, const float*, float*, int, cudaStream_t);

}  // namespace fno
