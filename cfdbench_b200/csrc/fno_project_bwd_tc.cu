// Backward of the project stage (fc1 -> GELU -> fc2 -> mask; reference src/models/fno/fno2d.py:228-233 under autograd,
// src/train_auto.py:255) on the tensor cores, both activation storage types.
//
// Per tile of 64 pixels (one image row), one warpgroup:
//   1. x tile -> tf32 hi / lo (bf16 storage: hi only, exact), K-major A operand; the loads of the NEXT tile are issued
//      before this tile's arithmetic.
//   2. GEMM1  z[64 px][128] = X W1^T           wgmma m64n128k8 tf32, 3xTF32 (2 passes in bf16 storage)
//   3. epilogue A (from the accumulator registers): z + b1 -> GELU and GELU' sharing one erfc;
//      dz = (w2[0] d0 + w2[1] d1) GELU'(z)  (d = dpreds * mask); dz goes to global memory (the fc1 weight gradient is
//      chan_outer's job) and, split into tf32 hi / lo, stays in registers as the A operand of GEMM2: the accumulator
//      fragment of a column pair (2 q, 2 q + 1) of a K = 8 block is exactly the A fragment of K positions (q, q + 4),
//      so the B operand of GEMM2 is stored with its K order permuted accordingly.  The pixel sums for the fc2 weight /
//      fc1 bias gradients use a halving transpose-reduction over the 8 lanes of a column, then fixed-order adds across
//      the four warps and across tiles.
//   4. GEMM2  da[64 px][32] = dz W1            wgmma m64n32k8 tf32 (register A), 3xTF32
//   5. epilogue B: da (x GELU'(pre) of the last Fourier block) -> d_out.
// Two warpgroup pipelines per CTA.  Deterministic: per-pipeline partial row [g_w2 256 | g_b1 128 | g_b2 2], reduced by
// reduce_partials in row order.
#include "../../include/cfdbench_b200.h"
#include "fno_common.cuh"
#include "tc_common.cuh"

namespace fno {

constexpr int kQbWG = 2;
constexpr int kQbThreads = 128 * kQbWG;
constexpr int kQbM = kW;                        // pixels per tile
constexpr int kQbTilesPerSample = kH;           // 64
constexpr int kQbOut = 3 * kProj + 2;           // partial row: g_w2 (2 x 128) | g_b1 (128) | g_b2 (2)
// Partial rows reserved for one launch: 16 per sample of a FNO_BWD_CHUNK batch chunk.  This sizes the caller's partial
// buffer (fno_bwd_partials_bytes()) and caps the grid; a cap below the SM count would change how many rows
// reduce_partials adds, and with it the last bits of the fc2.weight / fc1.bias / fc2.bias gradients.
constexpr int kQbRowsMax = 16 * FNO_BWD_CHUNK;
constexpr int kQbReps = kQbM * (kC / 4) / 128;  // 4 activation tasks per thread
constexpr uint32_t kQbLboA = (kQbM / 8) * 128;  // 1024
constexpr uint32_t kQbLboW1 = (kProj / 8) * 128;   // 2048
constexpr uint32_t kQbLboW1t = (kC / 8) * 128;     // 512

struct QbSmem {
  alignas(128) float w1_hi[kProj * kC];        // GEMM1 B operand: [n = hidden j][k = channel i] K-major
  alignas(128) float w1_lo[kProj * kC];
  alignas(128) float w1t_hi[kC * kProj];       // GEMM2 B operand: [n = channel i][k = hidden j, permuted] K-major
  alignas(128) float w1t_lo[kC * kProj];
  alignas(128) float x_hi[kQbWG][kQbM * kC];   // per pipeline
  alignas(128) float x_lo[kQbWG][kQbM * kC];
  alignas(16) float b1[kProj];
  alignas(16) float w2[2][kProj];
  alignas(16) float red[kQbWG][4][4][96];      // [pipeline][warp][lane % 4][kind * 32 + column]: per-warp pixel sums
  alignas(16) float acc[kQbWG][3 * kProj];     // running totals of a pipeline (fixed order: tile by tile)
  alignas(16) float red_b2[kQbWG][4][2];
};

__device__ __forceinline__ float qb_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// GELU and its derivative sharing one erfc evaluation
__device__ __forceinline__ void qb_gelu_both(float x, float& g, float& dg) {
  const float ax = fabsf(x);
  const float e = 0.5f * erfc_abs_scaled(ax);  // 0.5 erfc(|x|/sqrt2)
  g = fmaxf(x, 0.f) - ax * e;
  const float cdf = x >= 0.f ? 1.f - e : e;
  const float pdf = 0.3989422804014327f * ex2_approx(-0.7213475204444817f * x * x);
  dg = fmaf(x, pdf, cdf);
}

template <typename TAct>
__global__ void __launch_bounds__(kQbThreads, 1)
    project_bwd_tc_kernel(const TAct* __restrict__ a,         // [B][32][4096]  a_L
                          const float* __restrict__ dpreds,   // [B][2][4096]
                          const float* __restrict__ mask,     // [B][4096]
                          const float* __restrict__ pre,      // [B][32][4096] pre-activation of the last block (or null)
                          const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                          float* __restrict__ d_out,          // [B][32][4096]: dpre_{L-1} (pre != null) or d a_L
                          float* __restrict__ dz1,            // [B][128][4096]
                          float* __restrict__ partial,        // [pipeline][kQbOut]
                          int n_tiles) {
  constexpr bool kBf = sizeof(TAct) == 2;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  QbSmem& sm = *reinterpret_cast<QbSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tc::warp_index_uniform() >> 2, wq = (tid >> 5) & 3, t = tid & 127, q = lane & 3;

  // ---------------------------------------------------------------- prologue
  for (int e = tid; e < kProj * kC; e += kQbThreads) {   // w1[j][i]
    const int j = e / kC, i = e % kC;
    float hi, lo;
    tc::split_tf32(w1[e], hi, lo);
    const uint32_t o1 = tc::kmajor_offset(j, i, kProj) / 4;
    sm.w1_hi[o1] = hi;
    sm.w1_lo[o1] = lo;
    // K position of hidden unit j in GEMM2: block j / 8, position (j % 8) / 2 for even j, 4 + (j % 8) / 2 for odd j
    const int kk = (j & ~7) + ((j & 1) ? 4 + ((j & 7) >> 1) : ((j & 7) >> 1));
    const uint32_t o2 = tc::kmajor_offset(i, kk, kC) / 4;
    sm.w1t_hi[o2] = hi;
    sm.w1t_lo[o2] = lo;
  }
  for (int j = tid; j < kProj; j += kQbThreads) {
    sm.b1[j] = b1[j];
    sm.w2[0][j] = w2[j];
    sm.w2[1][j] = w2[kProj + j];
  }
  for (int e = tid; e < kQbWG * 3 * kProj; e += kQbThreads) (&sm.acc[0][0])[e] = 0.f;
  tc::fence_proxy_async_smem();   // the constant operands above are read by the tensor cores
  __syncthreads();

  const int first = blockIdx.x * kQbWG + wg, stride = gridDim.x * kQbWG;
  float* x_hi = sm.x_hi[wg];
  float* x_lo = sm.x_lo[wg];
  const int m0 = 16 * wq + (lane >> 2);   // fragment rows m0, m0 + 8
  TAct xr[kQbReps][4];   // task = rep * 128 + t -> (pixel m = task & 63, channel quad = task >> 6)
  auto x_load = [&](int tile) {
    const int b = tile / kQbTilesPerSample, p0 = (tile % kQbTilesPerSample) * kQbM;
#pragma unroll
    for (int rep = 0; rep < kQbReps; ++rep) {
      const int task = rep * 128 + t, m = task & (kQbM - 1), kq = task >> 6;
      const TAct* src = a + (static_cast<size_t>(b) * kC + 4 * kq) * kHW + p0 + m;
#pragma unroll
      for (int c = 0; c < 4; ++c) xr[rep][c] = __ldg(src + static_cast<size_t>(c) * kHW);
    }
  };
  if (first < n_tiles) x_load(first);
  float acc_b2[2] = {0.f, 0.f};   // sum over this thread's pixels of d0, d1 (lanes with lane % 4 == 0)

  for (int tile = first; tile < n_tiles; tile += stride) {
    const int b = tile / kQbTilesPerSample, p0 = (tile % kQbTilesPerSample) * kQbM;
    // ---- phase 1: x of this tile -> shared memory (the registers were loaded one tile ago)
#pragma unroll
    for (int rep = 0; rep < kQbReps; ++rep) {
      const int task = rep * 128 + t, m = task & (kQbM - 1), kq = task >> 6;
      float hi[4], lo[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float v = kBf ? __bfloat162float(xr[rep][c]) : static_cast<float>(xr[rep][c]);
        if constexpr (kBf) hi[c] = v;
        else tc::split_tf32(v, hi[c], lo[c]);
      }
      const uint32_t off = tc::kmajor_offset(m, 4 * kq, kQbM) / 4;
      *reinterpret_cast<float4*>(x_hi + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
      if constexpr (!kBf) *reinterpret_cast<float4*>(x_lo + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
    }
    tc::fence_proxy_async_smem();
    tc::named_barrier(1 + wg, 128);
    // ---- phase 2: GEMM1
    float z[64];
    tc::wg_fence();
    {
      const uint32_t a_s[3] = {tc::smem_addr(x_hi), tc::smem_addr(x_lo), tc::smem_addr(x_hi)};
      const uint32_t b_s[3] = {tc::smem_addr(sm.w1_hi), tc::smem_addr(sm.w1_hi), tc::smem_addr(sm.w1_lo)};
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {
        if (kBf && pass == 1) continue;
#pragma unroll
        for (int ks = 0; ks < kC / 8; ++ks)
          tc::wg_tf32_ss_n128(z, tc::make_smem_desc(a_s[pass] + ks * 2 * kQbLboA, kQbLboA, 128),
                              tc::make_smem_desc(b_s[pass] + ks * 2 * kQbLboW1, kQbLboW1, 128), (pass | ks) ? 1u : 0u);
      }
    }
    tc::wg_commit();
    if (tile + stride < n_tiles) x_load(tile + stride);
    float d[2][2];   // [row hh][out channel]
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int pix = p0 + m0 + 8 * hh;
      const float mk = __ldg(mask + static_cast<size_t>(b) * kHW + pix);
      d[hh][0] = __ldg(dpreds + (static_cast<size_t>(b) * 2 + 0) * kHW + pix) * mk;
      d[hh][1] = __ldg(dpreds + (static_cast<size_t>(b) * 2 + 1) * kHW + pix) * mk;
      if (q == 0) { acc_b2[0] += d[hh][0]; acc_b2[1] += d[hh][1]; }
    }
    tc::wg_wait<0>();
    tc::wg_fence_acc(z);
    // ---- phase 3: epilogue A.  z[4 i + 2 hh + e] = z[px = m0 + 8 hh][j = 8 i + 2 q + e], in four chunks of 4 i
    uint32_t dz_hi[16][4], dz_lo[16][4];   // GEMM2 A fragments: K block i, positions (q, q + 4) <-> j = 8 i + 2 q + (0, 1)
    float* dz_b = dz1 + static_cast<size_t>(b) * kProj * kHW + p0;
#pragma unroll
    for (int ic = 0; ic < 4; ++ic) {
      float v[24];   // [kind: d0 g | d1 g | dz][column c = 2 (i - 4 ic) + e], summed over the two rows
#pragma unroll
      for (int i = 4 * ic; i < 4 * ic + 4; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = 8 * i + 2 * q + e, c = 2 * (i - 4 * ic) + e;
          v[c] = v[8 + c] = v[16 + c] = 0.f;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float g, dg;
            qb_gelu_both(z[4 * i + 2 * hh + e] + sm.b1[j], g, dg);
            const float dz = (sm.w2[0][j] * d[hh][0] + sm.w2[1][j] * d[hh][1]) * dg;
            dz_b[static_cast<size_t>(j) * kHW + m0 + 8 * hh] = dz;
            float hi, lo;
            tc::split_tf32(dz, hi, lo);
            dz_hi[i][hh + 2 * e] = __float_as_uint(hi);   // a[0] = (r, q), a[1] = (r + 8, q), a[2] = (r, q + 4), a[3] = (r + 8, q + 4)
            dz_lo[i][hh + 2 * e] = __float_as_uint(lo);
            v[c] += d[hh][0] * g;
            v[8 + c] += d[hh][1] * g;
            v[16 + c] += dz;
          }
        }
      // halving transpose-reduction over the 8 lanes of a column (lane bits 4, 3, 2): 24 -> 12 -> 6 -> 3 values per lane
#pragma unroll
      for (int i = 0; i < 12; ++i) {
        const bool up = lane & 16;
        const float send = up ? v[i] : v[i + 12], keep = up ? v[i + 12] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
      }
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        const bool up = lane & 8;
        const float send = up ? v[i] : v[i + 6], keep = up ? v[i + 6] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const bool up = lane & 4;
        const float send = up ? v[i] : v[i + 3], keep = up ? v[i + 3] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
      const int off = ((lane >> 4) & 1) * 12 + ((lane >> 3) & 1) * 6 + ((lane >> 2) & 1) * 3;
#pragma unroll
      for (int i = 0; i < 3; ++i) sm.red[wg][wq][q][24 * ic + off + i] = v[i];
    }
    // ---- phase 4: GEMM2, da = dz W1 (A from registers); the pixel sums are added up while it runs
    float da[16];
    tc::wg_fence();
    {
      const uint32_t b_s[3] = {tc::smem_addr(sm.w1t_hi), tc::smem_addr(sm.w1t_hi), tc::smem_addr(sm.w1t_lo)};
#pragma unroll
      for (int pass = 0; pass < 3; ++pass)
#pragma unroll
        for (int ks = 0; ks < kProj / 8; ++ks)
          tc::wg_tf32_rs_n32(da, pass == 1 ? dz_lo[ks] : dz_hi[ks],
                             tc::make_smem_desc(b_s[pass] + ks * 2 * kQbLboW1t, kQbLboW1t, 128), (pass | ks) ? 1u : 0u);
    }
    tc::wg_commit();
    tc::named_barrier(1 + wg, 128);
    // running totals: entry (kind, hidden unit j) = sum over the four warps, in order
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int ent = r * 128 + t, kind = ent >> 7, j = ent & 127, i = j >> 3;
      const int qq = (j >> 1) & 3, idx = 24 * (i >> 2) + 8 * kind + 2 * (i & 3) + (j & 1);
      const float s = ((sm.red[wg][0][qq][idx] + sm.red[wg][1][qq][idx]) + sm.red[wg][2][qq][idx]) + sm.red[wg][3][qq][idx];
      sm.acc[wg][ent] += s;
    }
    // ---- phase 5: epilogue B.  da[4 i + 2 hh + e] = da[px = m0 + 8 hh][channel 8 i + 2 q + e]
    float pv[16];
    if (pre != nullptr) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            pv[4 * i + 2 * hh + e] =
                __ldg(pre + (static_cast<size_t>(b) * kC + 8 * i + 2 * q + e) * kHW + p0 + m0 + 8 * hh);
    }
    tc::wg_wait<0>();
    tc::wg_fence_acc(da);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float o = da[4 * i + 2 * hh + e];
          if (pre != nullptr) o *= dgelu_erf(pv[4 * i + 2 * hh + e]);
          d_out[(static_cast<size_t>(b) * kC + 8 * i + 2 * q + e) * kHW + p0 + m0 + 8 * hh] = o;
        }
  }
  // ---- the pipeline's partial row: [g_w2[0][j] | g_w2[1][j] | g_b1[j] | g_b2]
  {
    const float s0 = qb_warp_sum(acc_b2[0]), s1 = qb_warp_sum(acc_b2[1]);
    if (lane == 0) { sm.red_b2[wg][wq][0] = s0; sm.red_b2[wg][wq][1] = s1; }
  }
  tc::named_barrier(1 + wg, 128);
  float* prow = partial + static_cast<size_t>(blockIdx.x * kQbWG + wg) * kQbOut;
  for (int e = t; e < 3 * kProj; e += 128) prow[e] = sm.acc[wg][e];
  if (t < 2)
    prow[3 * kProj + t] = ((sm.red_b2[wg][0][t] + sm.red_b2[wg][1][t]) + sm.red_b2[wg][2][t]) + sm.red_b2[wg][3][t];
}

int project_bwd_rows_max() { return kQbRowsMax; }
int project_bwd_row() { return kQbOut; }

// returns the number of partial rows written through *n_parts
template <typename TAct>
cudaError_t launch_project_bwd_tc(const void* a, const float* dpreds, const float* mask, const float* pre, const float* w1,
                                  const float* b1, const float* w2, float* d_out, float* dz1, float* partial, int* n_parts,
                                  int batch, cudaStream_t stream) {
  auto kern = project_bwd_tc_kernel<TAct>;
  constexpr size_t smem = sizeof(QbSmem);
  static PerDeviceLaunch pd;
  int n_sm = 0;
  cudaError_t e0 = per_device_setup(kern, smem, pd, &n_sm);
  if (e0 != cudaSuccess) return e0;
  const int n_tiles = batch * kQbTilesPerSample;
  int grid = (n_tiles + kQbWG - 1) / kQbWG;
  if (grid > n_sm) grid = n_sm;
  if (grid > kQbRowsMax / kQbWG) grid = kQbRowsMax / kQbWG;   // the partial rows fit the caller's buffer
  kern<<<grid, kQbThreads, smem, stream>>>(static_cast<const TAct*>(a), dpreds, mask, pre, w1, b1, w2, d_out, dz1, partial, n_tiles);
  *n_parts = grid * kQbWG;
  return cudaGetLastError();
}
template cudaError_t launch_project_bwd_tc<float>(const void*, const float*, const float*, const float*, const float*, const float*,
                                                  const float*, float*, float*, float*, int*, int, cudaStream_t);
template cudaError_t launch_project_bwd_tc<__nv_bfloat16>(const void*, const float*, const float*, const float*, const float*,
                                                          const float*, const float*, float*, float*, float*, int*, int,
                                                          cudaStream_t);

}  // namespace fno
