// K1 on the tensor cores (bf16 activation storage) -- truncated forward 2-D DFT of activation planes:
//     x[b][c][64][64] (bf16)  ->  Xm[k][b][c]  (288 kept modes, complex64, mode-major).
//
// Replaces torch.fft.rfft2 + the two corner slices of the reference (src/models/fno/fno2d.py:62,73-78).
// Both 1-D transforms are GEMMs against constant twiddle matrices, on a unit of eight planes (one sample, channels
// 8 j .. 8 j + 7):
//
//  stage A (along w):  G_p[h][(q,ri)] = sum_w x_p[h][w] * TA[(q,ri)][w],  q = 0..11,  TA = (cos, -sin)(2 pi q w/64)
//      wgmma m64n72k16 bf16 per plane, K = 64.  The A operand IS the bf16 plane: TMA boxes {64 w, 128 rows} of two
//      planes land with the 128-byte swizzle as K-major operands, no register pass, exact.  TA is split into three bf16
//      terms (t1 + t2 + t3 carries 24 mantissa bits); the terms are column blocks of ONE N = 72 operand, ordered so that
//      the three terms of a column land in the same thread's accumulator registers, where they are added.  The sum is
//      stored in fp32 to the warpgroup's G buffer, row m = 16 q + 8 ri + p (td_g_index).
//  stage B (along h):  D[(q,ri,p)][(kxi,cs)] = sum_h G[(q,ri,p)][h] * T[(kxi,cs)][h],  T = (cos, sin)(2 pi kx h/64)
//      M = 192 (three m64 tiles), N = 48, K = 64; wgmma m64n48k8 tf32 as 3xTF32 with A from registers (each thread
//      splits its fragments of G into tf32 hi / lo) and the hi / lo images of T in shared memory.  Because x is real,
//      G[h][-q] = conj(G[h][q]): only q >= 0 is needed, and the 24 kept kx (0..11, 52..63) are T's 24 column pairs.
//  epilogue: the re and im rows of one (q, plane) are accumulator rows m0 and m0 + 8 of one thread and (kxi, cos) /
//      (kxi, sin) one column pair, so F_re = D[re][cos] + D[im][sin], F_im = D[im][cos] - D[re][sin] in registers; the
//      eight lanes of a row group hold the unit's eight planes of one mode: 64 contiguous bytes of Xm.
//
// Persistent CTA of two independent warpgroup pipelines, each with a TMA ring of kTdSlots two-plane boxes; a pipeline's
// fill n is box n % 4 of its unit n / 4 (td_slot, td_parity, td_box_row).
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
constexpr int kTdPlanes = 8;                                  // planes per unit
constexpr int kTdBoxPlanes = 2;                               // planes per TMA box
constexpr int kTdBoxes = kTdPlanes / kTdBoxPlanes;            // fills per unit
constexpr int kTdSlots = 3;                                   // ring depth per pipeline
constexpr uint32_t kTdPlaneBytes = kHW * 2;                   // 8,192 B
constexpr uint32_t kTdBoxBytes = kTdBoxPlanes * kTdPlaneBytes;  // 16,384 B
constexpr int kTdNA = 72;                                     // stage A N: 3 terms x 24
constexpr uint32_t kTdLboTA = (kTdNA / 8) * 128;              // 1152: K stride of the TA operand (8-element chunks)
constexpr uint32_t kTdTABytes = 8 * kTdLboTA;                 // 9,216 B
constexpr int kTdM2 = kM2 * 2 * kTdPlanes;                    // stage B M = 192: rows (q, ri, p)
constexpr int kTdN2 = 2 * kKX;                                // stage B N = 48: columns (kxi, cos | sin)
constexpr int kTdK2 = kH;                                     // stage B K = 64: h
constexpr uint32_t kTdLboT = (kTdN2 / 8) * 128;               // 768
constexpr int kTdTFloats = kTdN2 * kTdK2;                     // per image (hi or lo)
static_assert(kTdM2 == 3 * 64, "stage B is three full m64 tiles");

// Ring of one pipeline: fill n goes to slot n % kTdSlots and completes phase n / kTdSlots of that slot's barrier with
// kTdBoxBytes transaction bytes; its box starts at image row td_box_row(unit, n % kTdBoxes) of the [B*32*64][64] map.
__host__ __device__ constexpr int td_slot(int n) { return n % kTdSlots; }
__host__ __device__ constexpr uint32_t td_parity(int n) { return static_cast<uint32_t>(n / kTdSlots) & 1u; }
__host__ __device__ constexpr int td_box_row(int unit, int box) { return (unit * kTdPlanes + box * kTdBoxPlanes) * kH; }
// Unit i of pipeline `first` (stride = pipelines in the grid).
__host__ __device__ constexpr int td_unit(int first, int stride, int i) { return first + i * stride; }
__host__ __device__ constexpr int td_units_of(int first, int stride, int n_units) {
  return first < n_units ? (n_units - first + stride - 1) / stride : 0;
}
// fp32 G buffer [192][64]: row m = 16 q + 8 ri + p, column h XOR-swizzled so that both the stage-A stores (lanes over
// 8 h x 4 q) and the stage-B A-fragment loads (lanes over 8 p x 4 h) hit 32 distinct banks.
__host__ __device__ constexpr int td_g_index(int m, int h) {
  return m * kTdK2 + (h ^ (((m & 7) << 2) ^ (((m >> 4) & 3) << 3)));
}

struct TdSmem {
  alignas(1024) unsigned char x[kTdWG][kTdSlots][kTdBoxBytes];  // stage-A A operands (TMA, 128B swizzle)
  alignas(128) unsigned char ta[kTdTABytes];                    // stage-A B operand: three bf16 terms, K-major
  alignas(128) float t_hi[kTdTFloats];                          // stage-B B operand, K-major
  alignas(128) float t_lo[kTdTFloats];
  alignas(128) float g[kTdWG][kTdM2 * kTdK2];                   // stage-A result, stage-B A operand
  alignas(8) uint64_t x_full[kTdWG][kTdSlots];
};
static_assert(sizeof(TdSmem) <= 232448, "dft_fwd_tc_kernel exceeds the sm_90 opt-in shared memory");

__global__ void __launch_bounds__(kTdThreads, 1)
    dft_fwd_tc_kernel(const __grid_constant__ CUtensorMap x_map, float2* __restrict__ xm,
                      const unsigned char* __restrict__ ta_tab, const float* __restrict__ t_tab, int n_units, int batch,
                      float s0, float s1) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  TdSmem& sm = *reinterpret_cast<TdSmem*>(smem_raw);
  if ((smem_u32(smem_raw) & 1023u) != 0) __trap();
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tc::warp_index_uniform() >> 2, wq = (tid >> 5) & 3, t = tid & 127, q = lane & 3, lr = lane >> 2;
  const int first = blockIdx.x * kTdWG + wg, stride = gridDim.x * kTdWG;
  const int n_mine = td_units_of(first, stride, n_units);
  const int n_fills = n_mine * kTdBoxes;

  // ---------------------------------------------------------------- prologue (constant tables only)
  if (tid == 0) {
    for (int i = 0; i < kTdWG; ++i)
      for (int s = 0; s < kTdSlots; ++s) mbar_init(&sm.x_full[i][s], 1);
    fence_mbar_init();
  }
  for (int e = tid; e < static_cast<int>(kTdTABytes / 16); e += kTdThreads)
    reinterpret_cast<uint4*>(sm.ta)[e] = __ldg(reinterpret_cast<const uint4*>(ta_tab) + e);
  for (int e = tid; e < kTdTFloats / 4; e += kTdThreads) {
    reinterpret_cast<float4*>(sm.t_hi)[e] = __ldg(reinterpret_cast<const float4*>(t_tab) + e);
    reinterpret_cast<float4*>(sm.t_lo)[e] = __ldg(reinterpret_cast<const float4*>(t_tab + kTdTFloats) + e);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  pdl_wait();   // x comes from the previous kernel of the chain
  pdl_launch_dependents();

  auto load = [&](int n) {
    uint64_t* bar = &sm.x_full[wg][td_slot(n)];
    mbar_expect_tx(bar, kTdBoxBytes);
    tma_load_2d(sm.x[wg][td_slot(n)], &x_map, 0, td_box_row(td_unit(first, stride, n / kTdBoxes), n % kTdBoxes), bar);
  };
  if (t == 0)
    for (int n = 0; n < kTdSlots && n < n_fills; ++n) load(n);
  const int m0 = 16 * wq + lr;   // accumulator rows m0, m0 + 8
  const uint32_t ta_s = tc::smem_addr(sm.ta);
  float* g = sm.g[wg];
#pragma unroll 1
  for (int i = 0; i < n_mine; ++i) {
    // ---------------------------------------------------------------- stage A, two planes per fill
#pragma unroll 1
    for (int k = 0; k < kTdBoxes; ++k) {
      const int n = i * kTdBoxes + k;
      mbar_wait(&sm.x_full[wg][td_slot(n)], td_parity(n));
      float ga[kTdBoxPlanes][36];
      tc::wg_fence();
      const uint32_t x_s = tc::smem_addr(sm.x[wg][td_slot(n)]);
#pragma unroll
      for (int p = 0; p < kTdBoxPlanes; ++p)
#pragma unroll
        for (int ks = 0; ks < kW / 16; ++ks)   // K = 16 per MMA: 32 bytes inside the 128-byte swizzle row
          tc::wg_bf16_ss_n72(ga[p], tc::make_smem_desc_sw128(x_s + p * kTdPlaneBytes + ks * 32),
                             tc::make_smem_desc(ta_s + ks * 2 * kTdLboTA, kTdLboTA, 128), ks ? 1u : 0u);
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(ga[0]);
      tc::wg_fence_acc(ga[1]);
      if (t == 0 && n + kTdSlots < n_fills) load(n + kTdSlots);   // stage A has read the slot
      if (k == 0) tc::named_barrier(1 + wg, 128);   // every thread has loaded the previous unit's G (stage B)
      // ga[p][4 (3 g + term) + 2 hh + ri] = G_p[h = m0 + 8 hh][q = 4 g + lane % 4][ri], term 0..2 (TA row order, see
      // td_ensure) -> G[16 q + 8 ri + plane][h]
#pragma unroll
      for (int p = 0; p < kTdBoxPlanes; ++p)
#pragma unroll
        for (int g3 = 0; g3 < 3; ++g3)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ri = 0; ri < 2; ++ri) {
              const int c = 4 * (3 * g3) + 2 * hh + ri;
              g[td_g_index(16 * (4 * g3 + q) + 8 * ri + kTdBoxPlanes * k + p, m0 + 8 * hh)] =
                  (ga[p][c + 8] + ga[p][c + 4]) + ga[p][c];
            }
    }
    tc::named_barrier(1 + wg, 128);   // G is complete
    // ---------------------------------------------------------------- stage B + epilogue, one m64 tile (4 q) at a time
    const int unit = td_unit(first, stride, i);
    const int b = unit * kTdPlanes / kC, c0 = unit * kTdPlanes % kC;
#pragma unroll 1
    for (int tile = 0; tile < kTdM2 / 64; ++tile) {
      // A fragment of k-step ks: rows m0 (re), m0 + 8 (im) of the tile, columns h = 8 ks + lane % 4 (+ 4)
      uint32_t a_hi[kTdK2 / 8][4], a_lo[kTdK2 / 8][4];
#pragma unroll
      for (int ks = 0; ks < kTdK2 / 8; ++ks)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float hi, lo;
          tc::split_tf32(g[td_g_index(64 * tile + m0 + 8 * (r & 1), 8 * ks + q + 4 * (r >> 1))], hi, lo);
          a_hi[ks][r] = __float_as_uint(hi);
          a_lo[ks][r] = __float_as_uint(lo);
        }
      float d[24];
      tc::wg_fence();
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {   // A_hi x T_hi, A_hi x T_lo, A_lo x T_hi
        const uint32_t tb = tc::smem_addr(pass == 1 ? sm.t_lo : sm.t_hi);
#pragma unroll
        for (int ks = 0; ks < kTdK2 / 8; ++ks)
          tc::wg_tf32_rs_n48(d, pass == 2 ? a_lo[ks] : a_hi[ks], tc::make_smem_desc(tb + ks * 2 * kTdLboT, kTdLboT, 128),
                             (pass | ks) ? 1u : 0u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc(d);
      // d[4 j + 2 ri + cs] = D[(q = 4 tile + wq, ri, plane = lane / 4)][(kxi = 4 j + lane % 4, cs)]
      const int qq = 4 * tile + wq;
      const float sc = qq == 0 ? s0 : s1;
#pragma unroll
      for (int j = 0; j < kTdN2 / 8; ++j) {
        const int kxi = 4 * j + q;
        const float re = (d[4 * j + 0] + d[4 * j + 3]) * sc, im = (d[4 * j + 2] - d[4 * j + 1]) * sc;
        xm[(static_cast<size_t>(kxi * kM2 + qq) * batch + b) * kC + c0 + lr] = make_float2(re, im);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Constant tables, built once per device from float64:
//   TA  -- three bf16 terms of (cos, -sin)(2 pi q w / 64) as ONE K-major operand of 72 rows: term t of column (q, ri) is
//          row 8 (3 (q / 4) + t) + 2 (q % 4) + ri, i.e. the accumulator registers 4 (3 (q / 4) + t) + 2 hh + ri of the
//          thread with lane % 4 = q % 4 (fragment layout in tc_common.cuh).
//   T   -- [n = 2 kxi + cs][h] = (cos, sin)(2 pi kx h / 64) as tf32 hi image | lo image, K-major.
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

struct TdTables {
  unsigned char* ta = nullptr;
  float* t = nullptr;
  int n_sm = 0;
  bool configured = false;
};
static TdTables g_td[64];

static cudaError_t td_ensure(int dev, cudaStream_t stream) {
  TdTables& t = g_td[dev];
  if (t.configured) return cudaSuccess;
  static unsigned char h_ta[kTdTABytes];
  static float h_t[2 * kTdTFloats];
  memset(h_ta, 0, sizeof(h_ta));
  memset(h_t, 0, sizeof(h_t));
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
    for (int cs = 0; cs < 2; ++cs)
      for (int h = 0; h < kH; ++h) {
        const double ang = two_pi * ((kx * h) % 64) / 64.0;
        const double val = cs ? sin(ang) : cos(ang);
        const uint32_t off = tc::kmajor_offset(2 * kxi + cs, h, kTdN2) / 4;
        const float hi = tc::round_tf32(static_cast<float>(val));
        h_t[off] = hi;
        h_t[kTdTFloats + off] = tc::round_tf32(static_cast<float>(val - static_cast<double>(hi)));
      }
  }
  cudaError_t e = cudaMalloc(&t.ta, sizeof(h_ta));
  if (e != cudaSuccess) return e;
  e = cudaMalloc(&t.t, sizeof(h_t));
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(t.ta, h_ta, sizeof(h_ta), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(t.t, h_t, sizeof(h_t), cudaMemcpyHostToDevice, stream);
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
  if (t.t) cudaFree(t.t);
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
                      kTdBoxPlanes * kH);
  if (e != cudaSuccess) return e;
  const int n_units = batch * kC / kTdPlanes;
  // the fewest CTAs that keep the busiest pipeline at ceil(n_units / (2 SMs)) units: the same finish time, and the
  // SMs left over take the next kernel's CTAs early (programmatic dependent launch)
  const int per_pipe = (n_units + kTdWG * g_td[dev].n_sm - 1) / (kTdWG * g_td[dev].n_sm);
  const int grid = (n_units + kTdWG * per_pipe - 1) / (kTdWG * per_pipe);
  return launch_chained(dft_fwd_tc_kernel, dim3(grid), dim3(kTdThreads), sizeof(TdSmem), stream, map,
                        static_cast<float2*>(xm), static_cast<const unsigned char*>(g_td[dev].ta),
                        static_cast<const float*>(g_td[dev].t), n_units, batch, s0, s1);
}

}  // namespace fno
