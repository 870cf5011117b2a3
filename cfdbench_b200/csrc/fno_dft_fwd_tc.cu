// K1 on the tensor cores (bf16 activation storage) -- truncated forward 2-D DFT of activation planes:
//     x[b][c][64][64] (bf16)  ->  Xm[k][b][c]  (288 kept modes, complex64, mode-major).
//
// Replaces torch.fft.rfft2 + the two corner slices of the reference (src/models/fno/fno2d.py:62,73-78).
// Both 1-D transforms are GEMMs against constant twiddle matrices, on a pair of planes (one sample, two channels):
//
//  stage A (along w):  G_p[h][(q,ri)] = sum_w x_p[h][w] * TA[(q,ri)][w],  q = 0..11,  TA = (cos, -sin)(2 pi q w/64)
//      wgmma m64n72k16 bf16 per plane, K = 64.  The A operand IS the bf16 plane: one TMA box {64 w, 128 rows} with the
//      128-byte swizzle lands both planes as K-major operands, no register pass, exact.  TA is split into three bf16 terms
//      (t1 + t2 + t3 carries 24 mantissa bits); the terms are column blocks of ONE N = 72 operand, ordered so that the
//      three terms of a column land in the same thread's accumulator registers, where they are added.
//  stage B (along h):  F[(kxi,part)][(q,p)] = sum_{(ri,h)} A2[(kxi,part)][(ri,h)] * G_p[h][q][ri],  kxi = 0..23
//      wgmma m64n24k8 tf32 as 3xTF32, K = 128; A2 = (c, s | -s, c) is a constant (48 rows, padded to 64) kept in shared
//      memory for the whole kernel; the B operand is stage A's result, summed over the terms, split into tf32 hi / lo and
//      written K-major.  Because x is real, G[h][-q] = conj(G[h][q]): only q >= 0 is computed and stage B produces all
//      24 kept kx rows (kx = 0..11 and 52..63) of the 12 kept columns directly.
//  epilogue: pairs the (kxi,re) / (kxi,im) rows (lane ^ 4) and writes (re, im) of one plane per lane.
//
// Persistent CTA of two independent warpgroup pipelines, each with a two-slot TMA ring of plane pairs.
// The register-FFT kernel (fno_dft_fwd.cu) remains for fp32 storage and the fp32 gradients of the backward pass.
#include "fno_common.cuh"
#include "tc_common.cuh"
#include "tc_tma.cuh"
#include <math.h>
#include <stddef.h>
#include <string.h>

namespace fno {

constexpr int kTdWG = 2;
constexpr int kTdThreads = 128 * kTdWG;
constexpr int kTdPlanes = 2;                               // planes per unit
constexpr uint32_t kTdPlaneBytes = kHW * 2;                // 8,192 B
constexpr uint32_t kTdXBytes = kTdPlanes * kTdPlaneBytes;  // 16,384 B per unit
constexpr int kTdNA = 72;                                  // stage A N: 3 terms x 24
constexpr uint32_t kTdLboTA = (kTdNA / 8) * 128;           // 1152: K stride of the TA operand (8-element chunks)
constexpr uint32_t kTdTABytes = 8 * kTdLboTA;              // 9,216 B
constexpr int kTdK2 = 128, kTdN2 = kTdPlanes * kM2;        // stage B: K = (ri, h), N = 24, column n2 = 2 q + p
constexpr int kTdM2 = 64;                                  // stage B rows (48 used)
constexpr uint32_t kTdLboA2 = (kTdM2 / 8) * 128;           // 1024
constexpr uint32_t kTdLboB2 = (kTdN2 / 8) * 128;           // 384
constexpr int kTdA2Floats = kTdM2 * kTdK2;                 // per image (hi or lo)

struct TdSmem {
  alignas(1024) unsigned char x[kTdWG][2][kTdXBytes];   // stage-A A operands (TMA, 128B swizzle): [pipeline][slot]
  alignas(128) unsigned char ta[kTdTABytes];            // stage-A B operand: three bf16 terms, K-major
  alignas(128) float a2_hi[kTdA2Floats];                // stage-B A operand, K-major
  alignas(128) float a2_lo[kTdA2Floats];
  alignas(128) float b2[kTdWG][2][kTdN2 * kTdK2];       // stage-B B operand: [pipeline][tf32 hi, lo]
  alignas(8) uint64_t x_full[kTdWG][2];
};

__global__ void __launch_bounds__(kTdThreads, 1)
    dft_fwd_tc_kernel(const __grid_constant__ CUtensorMap x_map, float2* __restrict__ xm,
                      const unsigned char* __restrict__ ta_tab, const float* __restrict__ a2_tab, int n_units, int batch,
                      float s0, float s1) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  TdSmem& sm = *reinterpret_cast<TdSmem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tc::warp_index_uniform() >> 2, wq = (tid >> 5) & 3, t = tid & 127, q = lane & 3;
  const int first = blockIdx.x * kTdWG + wg, stride = gridDim.x * kTdWG;
  const int n_mine = first < n_units ? (n_units - first + stride - 1) / stride : 0;

  // ---------------------------------------------------------------- prologue (constant tables only)
  if (tid == 0) {
    for (int i = 0; i < kTdWG; ++i) { mbar_init(&sm.x_full[i][0], 1); mbar_init(&sm.x_full[i][1], 1); }
    fence_mbar_init();
  }
  for (int e = tid; e < static_cast<int>(kTdTABytes / 16); e += kTdThreads)
    reinterpret_cast<uint4*>(sm.ta)[e] = __ldg(reinterpret_cast<const uint4*>(ta_tab) + e);
  for (int e = tid; e < kTdA2Floats / 4; e += kTdThreads) {
    reinterpret_cast<float4*>(sm.a2_hi)[e] = __ldg(reinterpret_cast<const float4*>(a2_tab) + e);
    reinterpret_cast<float4*>(sm.a2_lo)[e] = __ldg(reinterpret_cast<const float4*>(a2_tab + kTdA2Floats) + e);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  pdl_wait();   // x comes from the previous kernel of the chain
  pdl_launch_dependents();

  auto load = [&](int i) {   // unit i of this pipeline -> slot i & 1
    mbar_expect_tx(&sm.x_full[wg][i & 1], kTdXBytes);
    tma_load_2d(sm.x[wg][i & 1], &x_map, 0, (first + i * stride) * (kTdPlanes * kH), &sm.x_full[wg][i & 1]);
  };
  if (t == 0) {
    if (n_mine > 0) load(0);
    if (n_mine > 1) load(1);
  }
  const int m0 = 16 * wq + (lane >> 2);   // accumulator rows m0, m0 + 8
  const uint32_t ta_s = tc::smem_addr(sm.ta);
  float* b2_hi = sm.b2[wg][0];
  float* b2_lo = sm.b2[wg][1];
#pragma unroll 1
  for (int i = 0; i < n_mine; ++i) {
    const int s = i & 1;
    mbar_wait(&sm.x_full[wg][s], (i >> 1) & 1);
    // ---------------------------------------------------------------- stage A
    float ga[kTdPlanes][36];
    tc::wg_fence();
    const uint32_t x_s = tc::smem_addr(sm.x[wg][s]);
#pragma unroll
    for (int p = 0; p < kTdPlanes; ++p)
#pragma unroll
      for (int ks = 0; ks < kW / 16; ++ks)   // K = 16 per MMA: 32 bytes inside the 128-byte swizzle row
        tc::wg_bf16_ss_n72(ga[p], tc::make_smem_desc_sw128(x_s + p * kTdPlaneBytes + ks * 32),
                           tc::make_smem_desc(ta_s + ks * 2 * kTdLboTA, kTdLboTA, 128), ks ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_fence_acc(ga[0]);
    tc::wg_fence_acc(ga[1]);
    if (t == 0 && i + 2 < n_mine) load(i + 2);   // stage A has read the slot
    // ga[p][4 (3 g + term) + 2 hh + ri] = G_p[h = m0 + 8 hh][q = 4 g + lane % 4][ri], term 0..2 (TA row order, see td_ensure)
    // -> B2[n2 = 2 q + p][k2 = 64 ri + h], tf32 hi / lo.  Stage B of the previous unit is complete (waited for below).
#pragma unroll
    for (int p = 0; p < kTdPlanes; ++p)
#pragma unroll
      for (int g3 = 0; g3 < 3; ++g3)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int ri = 0; ri < 2; ++ri) {
            const int c = 4 * (3 * g3) + 2 * hh + ri;
            const float gsum = (ga[p][c + 8] + ga[p][c + 4]) + ga[p][c];
            float hi, lo;
            tc::split_tf32(gsum, hi, lo);
            const uint32_t off = tc::kmajor_offset(2 * (4 * g3 + q) + p, 64 * ri + m0 + 8 * hh, kTdN2) / 4;
            b2_hi[off] = hi;
            b2_lo[off] = lo;
          }
    tc::fence_proxy_async_smem();
    tc::named_barrier(1 + wg, 128);
    // ---------------------------------------------------------------- stage B
    float fb[12];
    tc::wg_fence();
    {
      const uint32_t a_s[3] = {tc::smem_addr(sm.a2_hi), tc::smem_addr(sm.a2_lo), tc::smem_addr(sm.a2_hi)};
      const uint32_t b_s[3] = {tc::smem_addr(b2_hi), tc::smem_addr(b2_hi), tc::smem_addr(b2_lo)};
#pragma unroll
      for (int pass = 0; pass < 3; ++pass)
#pragma unroll
        for (int ks = 0; ks < kTdK2 / 8; ++ks)
          tc::wg_tf32_ss_n24(fb, tc::make_smem_desc(a_s[pass] + ks * 2 * kTdLboA2, kTdLboA2, 128),
                             tc::make_smem_desc(b_s[pass] + ks * 2 * kTdLboB2, kTdLboB2, 128), (pass | ks) ? 1u : 0u);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_fence_acc(fb);
    // ---------------------------------------------------------------- epilogue
    // fb[4 j + 2 hh + p] = F[m2 = m0 + 8 hh = 2 kxi + part][q = 4 j + lane % 4][plane p]; lane ^ 4 holds the other part
    const int part = (lane >> 2) & 1;
    const int plane0 = (first + i * stride) * kTdPlanes;
    const int b = plane0 / kC, c0 = plane0 % kC;
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int qq = 4 * j + q, m2 = m0 + 8 * hh, kxi = m2 >> 1;
        const float sc = qq == 0 ? s0 : s1;
        const float v0 = fb[4 * j + 2 * hh] * sc, v1 = fb[4 * j + 2 * hh + 1] * sc;
        // the re lane keeps plane 0 and needs its im; the im lane keeps plane 1 and needs its re
        const float got = __shfl_xor_sync(0xffffffffu, part ? v0 : v1, 4);
        if (m2 < 2 * kKX) {
          float2* dst = xm + (static_cast<size_t>(kxi * kM2 + qq) * batch + b) * kC + c0 + part;
          *dst = part ? make_float2(got, v1) : make_float2(v0, got);
        }
      }
  }
}

// ------------------------------------------------------------------------------------------------
// Constant tables, built once per device from float64:
//   TA  -- three bf16 terms of (cos, -sin)(2 pi q w / 64) as ONE K-major operand of 72 rows: term t of column (q, ri) is
//          row 8 (3 (q / 4) + t) + 2 (q % 4) + ri, i.e. the accumulator registers 4 (3 (q / 4) + t) + 2 hh + ri of the
//          thread with lane % 4 = q % 4 (fragment layout in tc_common.cuh).
//   A2  -- [m2 = 2 kxi + part (64, rows 48..63 zero)][k2 = ri*64 + h] as tf32 hi image | lo image, K-major.
// ------------------------------------------------------------------------------------------------
static uint16_t td_bf16_bits(double v) {  // round to nearest even
  float f = static_cast<float>(v);
  uint32_t u;
  memcpy(&u, &f, 4);
  const uint32_t r = u + 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(r >> 16);
}
static double td_bf16_value(uint16_t b) {
  const uint32_t u = static_cast<uint32_t>(b) << 16;
  float f;
  memcpy(&f, &u, 4);
  return static_cast<double>(f);
}
static float td_round_tf32(double v) {
  float f = static_cast<float>(v);
  uint32_t u;
  memcpy(&u, &f, 4);
  u = (u + 0x1000u) & 0xffffe000u;
  memcpy(&f, &u, 4);
  return f;
}

struct TdTables {
  unsigned char* ta = nullptr;
  float* a2 = nullptr;
  int n_sm = 0;
  bool configured = false;
};
static TdTables g_td[64];

static cudaError_t td_ensure(int dev, cudaStream_t stream) {
  TdTables& t = g_td[dev];
  if (t.configured) return cudaSuccess;
  static unsigned char h_ta[kTdTABytes];
  static float h_a2[2 * kTdA2Floats];
  memset(h_ta, 0, sizeof(h_ta));
  memset(h_a2, 0, sizeof(h_a2));
  const double two_pi = 2.0 * 3.14159265358979323846;
  for (int q = 0; q < kM2; ++q)
    for (int ri = 0; ri < 2; ++ri)
      for (int w = 0; w < 64; ++w) {
        const double ang = two_pi * ((q * w) % 64) / 64.0;
        double rest = ri ? -sin(ang) : cos(ang);
        for (int t3 = 0; t3 < 3; ++t3) {
          const int row = 8 * (3 * (q >> 2) + t3) + 2 * (q & 3) + ri;
          const size_t off = static_cast<size_t>(w >> 3) * kTdLboTA + (row >> 3) * 128 + (row & 7) * 16 + (w & 7) * 2;
          const uint16_t bits = td_bf16_bits(rest);
          memcpy(h_ta + off, &bits, 2);
          rest -= td_bf16_value(bits);
        }
      }
  for (int kxi = 0; kxi < kKX; ++kxi) {
    const int kx = kxi < kM1 ? kxi : kxi + (kH - kKX);
    for (int part = 0; part < 2; ++part)
      for (int ri = 0; ri < 2; ++ri)
        for (int h = 0; h < 64; ++h) {
          const double ang = two_pi * ((kx * h) % 64) / 64.0;
          const double c = cos(ang), s = sin(ang);
          // Fre = sum c Gre + s Gim;  Fim = sum -s Gre + c Gim
          const double val = part == 0 ? (ri == 0 ? c : s) : (ri == 0 ? -s : c);
          const uint32_t off = tc::kmajor_offset(2 * kxi + part, ri * 64 + h, kTdM2) / 4;
          const float hi = td_round_tf32(val);
          h_a2[off] = hi;
          h_a2[kTdA2Floats + off] = td_round_tf32(val - static_cast<double>(hi));
        }
  }
  cudaError_t e = cudaMalloc(&t.ta, sizeof(h_ta));
  if (e != cudaSuccess) return e;
  e = cudaMalloc(&t.a2, sizeof(h_a2));
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(t.ta, h_ta, sizeof(h_ta), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(t.a2, h_a2, sizeof(h_a2), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) return e;
  e = cudaStreamSynchronize(stream);   // the host arrays are static
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(dft_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TdSmem));
  if (e != cudaSuccess) return e;
  e = cudaDeviceGetAttribute(&t.n_sm, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  t.configured = true;
  return cudaSuccess;
}

void dft_fwd_tc_release(int dev) {
  if (dev < 0 || dev >= 64) return;
  TdTables& t = g_td[dev];
  if (t.ta) cudaFree(t.ta);
  if (t.a2) cudaFree(t.a2);
  t = TdTables();
}

cudaError_t launch_dft_fwd_tc(const void* x, void* xm, int batch, float s0, float s1, cudaStream_t stream) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  e = td_ensure(dev, stream);
  if (e != cudaSuccess) return e;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(xm) & 15)) return cudaErrorMisalignedAddress;
  // a bf16 activation seen as rows of one image row each: [batch * 32 * 64 rows][64 w], box {64, 128} = two planes
  CUtensorMap map;
  e = make_tma_map_2d(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, kW, static_cast<uint64_t>(batch) * kC * kH, kW,
                      kTdPlanes * kH);
  if (e != cudaSuccess) return e;
  const int n_units = batch * kC / kTdPlanes;
  const int want = (n_units + kTdWG - 1) / kTdWG;
  const int grid = want < g_td[dev].n_sm ? want : g_td[dev].n_sm;
  return launch_chained(dft_fwd_tc_kernel, dim3(grid), dim3(kTdThreads), sizeof(TdSmem), stream, map,
                        static_cast<float2*>(xm), static_cast<const unsigned char*>(g_td[dev].ta),
                        static_cast<const float*>(g_td[dev].a2), n_units, batch, s0, s1);
}

}  // namespace fno
