// Fourier-block output stage on the tensor cores (K3 = K3a + K3b):
//   out[b][o][h][w] = act( irfft2(pad(Y))[b][o][h][w] + sum_i W0[o][i] x[b][i][h][w] + bias[o] )
// replacing irfft2 + Conv2d(32,32,1) + add + GELU of the reference FnoBlock
// (src/models/fno/fno2d.py:65-72,81,104-111).
//
// K3a  inv_kx_kernel   inverse DFT along kx of the 24 kept rows (codelet icfft64_in24_full, one thread per
//                      (ky, o)), scaled by c_ky/HW, written as Z[b][h][k][o], k = 2 ky + (re|im): 196 KB/sample.
// K3b  block_tc_kernel per image row: the C2R stage along w and the 1x1 convolution as one wgmma accumulation chain
//                      (below), epilogue GELU (or the backward epilogues) from the accumulator registers.
#include "fft_codelets.cuh"
#include "fno_common.cuh"
#include "tc_common.cuh"
#include <math.h>
#include <stddef.h>
#include <string.h>

namespace fno {

enum : int { kEpiGelu = 0, kEpiGeluSavePre = 1, kEpiMulDgelu = 2, kEpiPlain = 3 };

// ------------------------------------------------------------------------------------------------ K3a
constexpr int kIkThreads = 192;  // 6 ky x 32 o per CTA, 2 CTAs per sample
constexpr int kZK = 2 * kM2;     // 24 real columns per row: (ky, re|im)

__global__ void __launch_bounds__(kIkThreads)
    inv_kx_kernel(const float2* __restrict__ ym, float* __restrict__ z, float s0, float s1) {
  const int b = blockIdx.y;
  const int ky = blockIdx.x * (kIkThreads / 32) + (threadIdx.x >> 5);
  const int o = threadIdx.x & 31;
  const float2* ym_b = ym + static_cast<size_t>(b) * kC;             // modes are stored mode-major: ym[k][b][o]
  const size_t mode_stride = static_cast<size_t>(gridDim.y) * kC;   // batch * 32
  float yre[kKX], yim[kKX], ore[kH], oim[kH];
  pdl_wait();
  pdl_launch_dependents();
#pragma unroll
  for (int kxi = 0; kxi < kKX; ++kxi) {
    const float2 v = __ldg(ym_b + (kxi * kM2 + ky) * mode_stride + o);
    yre[kxi] = v.x;
    yim[kxi] = v.y;
  }
  fno_codelets::icfft64_in24_full<float>(yre, yim, ore, oim);
  const float s = (ky == 0) ? s0 : s1;
  float* zb = z + (static_cast<size_t>(b) * kH * kZK + 2 * ky) * kC + o;
#pragma unroll
  for (int h = 0; h < kH; ++h) {
    zb[static_cast<size_t>(h) * kZK * kC] = ore[h] * s;
    zb[static_cast<size_t>(h) * kZK * kC + kC] = oim[h] * s;
  }
}

cudaError_t launch_inv_kx(const void* ym, void* z, int batch, float s0, float s1, cudaStream_t stream) {
  dim3 grid(kM2 / (kIkThreads / 32), batch);
  return launch_chained<false>(inv_kx_kernel, grid, dim3(kIkThreads), 0, stream, static_cast<const float2*>(ym),
                        static_cast<float*>(z), s0, s1);
}

// ------------------------------------------------------------------------------------------------ K3b
constexpr int kBtWG = 4;                       // independent warpgroup pipelines per CTA
constexpr int kBtThreads = 128 * kBtWG;
constexpr int kBtM = kW;                       // pixels per tile: one image row
constexpr int kKE = kZK;                       // 24: E-part K
constexpr int kKConv = kC;                     // 32: conv-part K
constexpr uint32_t kLboA = (kBtM / 8) * 128;   // 1024
constexpr uint32_t kLboB = (kC / 8) * 128;     // 512
constexpr int kBtTilesPerSample = kH;          // 64
constexpr int kETabFloats = 2 * kBtM * kKE;    // hi image, then lo image
constexpr int kBtXReps = kBtM * (kKConv / 4) / 128;   // 4 x-tasks per thread
constexpr int kBtZTasks = kC * (kKE / 4);             // 192
static_assert(2 * 128 >= kBtZTasks, "two z reps must cover the tile");

struct BtSmem {
  alignas(128) float e_hi[kBtM * kKE];              // A operand, E part (constant)       6,144 B
  alignas(128) float e_lo[kBtM * kKE];
  alignas(128) float wb_hi[kC * kKConv];            // B operand, conv part               4,096 B
  alignas(128) float wb_lo[kC * kKConv];
  alignas(128) float ax_hi[kBtWG][kBtM * kKConv];   // A operand, conv part, per pipeline 8,192 B
  alignas(128) float ax_lo[kBtWG][kBtM * kKConv];
  alignas(128) float bz_hi[kBtWG][kC * kKE];        // B operand, E part, per pipeline    3,072 B
  alignas(128) float bz_lo[kBtWG][kC * kKE];
  alignas(16) float bias[kC];
};

template <typename TAct>
struct BtRegs {
  TAct x[kBtXReps][4];  // task = rep*128 + t -> (pixel m = task & 63, channel quad = task >> 6)
  float z[2][4];        // task = rep*128 + t (< 192) -> (o = task & 31, k quad = task >> 5)
};

__device__ __forceinline__ float bt_to_float(float v) { return v; }
__device__ __forceinline__ float bt_to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ void bt_store(float* p, float v) { *p = v; }
__device__ __forceinline__ void bt_store(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

template <typename TAct>
__device__ __forceinline__ void bt_prefetch(BtRegs<TAct>& r, const TAct* __restrict__ x, const float* __restrict__ z,
                                            int tile, int t) {
  const int b = tile / kBtTilesPerSample, h = tile % kBtTilesPerSample;
#pragma unroll
  for (int rep = 0; rep < kBtXReps; ++rep) {
    const int task = rep * 128 + t;
    const int m = task & (kBtM - 1), kq = task >> 6;
    const TAct* src = x + (static_cast<size_t>(b) * kC + 4 * kq) * kHW + h * kW + m;
#pragma unroll
    for (int c = 0; c < 4; ++c) r.x[rep][c] = __ldg(src + static_cast<size_t>(c) * kHW);
  }
#pragma unroll
  for (int rep = 0; rep < 2; ++rep) {
    const int task = rep * 128 + t;
    if (task < kBtZTasks) {
      const int o = task & 31, kq = task >> 5;
      const float* src = z + ((static_cast<size_t>(b) * kH + h) * kZK + 4 * kq) * kC + o;
#pragma unroll
      for (int c = 0; c < 4; ++c) r.z[rep][c] = __ldg(src + c * kC);
    }
  }
}

template <typename TAct>
__device__ __forceinline__ void bt_split_store(const BtRegs<TAct>& r, float* ax_hi, float* ax_lo, float* bz_hi,
                                               float* bz_lo, const float* bias_s, int t) {
#pragma unroll
  for (int rep = 0; rep < kBtXReps; ++rep) {
    const int task = rep * 128 + t;
    const int m = task & (kBtM - 1), kq = task >> 6;
    float hi[4], lo[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float v = bt_to_float(r.x[rep][c]);
      if constexpr (sizeof(TAct) == 4) tc::split_tf32(v, hi[c], lo[c]);
      else hi[c] = v;  // bf16 is tf32-exact: no lo part
    }
    const uint32_t off = tc::kmajor_offset(m, 4 * kq, kBtM) / 4;
    *reinterpret_cast<float4*>(ax_hi + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
    if constexpr (sizeof(TAct) == 4) *reinterpret_cast<float4*>(ax_lo + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
  }
#pragma unroll
  for (int rep = 0; rep < 2; ++rep) {
    const int task = rep * 128 + t;
    if (task < kBtZTasks) {
      const int o = task & 31, kq = task >> 5;
      float hi[4], lo[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float v = r.z[rep][c];
        // K column 1 (Im of the ky = 0 column, which the C2R stage ignores) carries the bias instead: the E table holds 1
        // there, so the MMA adds bias[o] to every pixel.
        if (c == 1 && kq == 0) v = bias_s[o];
        tc::split_tf32(v, hi[c], lo[c]);
      }
      const uint32_t off = tc::kmajor_offset(o, 4 * kq, kC) / 4;
      *reinterpret_cast<float4*>(bz_hi + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<float4*>(bz_lo + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
    }
  }
}

// K3b: per tile (one image row of one sample, 64 pixels) one warpgroup runs the accumulation chain
//     D[64 px][32 o] = [E | X] * [Z_h ; W0^T]        K = 24 + 32, wgmma m64n32k8 tf32, 3xTF32
// E[w][k] = (cos, -sin)(2 pi ky w/64) is the C2R stage of the inverse transform as a constant matrix (its ky=0 imaginary
// column would be zero -- irfft2 drops Im of the DC column -- and carries the bias instead: E = 1 there, the B row = bias).
// Four independent warpgroup pipelines per CTA; a pipeline prefetches the next tile's operands into registers while the
// current tile's MMAs and epilogue run, splits them into tf32 hi/lo (round-to-nearest) and writes them as K-major operands.
template <typename TAct, int EPI>
__global__ void __launch_bounds__(kBtThreads, 1)
    block_tc_kernel(const float* __restrict__ z, const TAct* __restrict__ x, const float* __restrict__ w0t,
                    const float* __restrict__ bias, const float* __restrict__ etab, TAct* __restrict__ out,
                    float* __restrict__ pre_out, const float* __restrict__ pre_in, int n_tiles) {
  constexpr bool kBf16 = sizeof(TAct) == 2;
  extern __shared__ __align__(1024) unsigned char smem_raw[];  // no pointer arithmetic: keeps LDS/STS addressing
  BtSmem& sm = *reinterpret_cast<BtSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tc::warp_index_uniform() >> 2, t = tid & 127, wq = (tid >> 5) & 3;

  static_assert(offsetof(BtSmem, e_lo) == offsetof(BtSmem, e_hi) + kETabFloats * 2, "e_hi / e_lo must be contiguous");
  for (int e = tid; e < kETabFloats; e += kBtThreads) sm.e_hi[e] = __ldg(etab + e);   // runs on into e_lo
  for (int e = tid; e < kC * kKConv; e += kBtThreads) {  // B[n = o][k = i] = W0[o][i] = w0t[i][o]
    const int i = e / kC, o = e % kC;
    float hi, lo;
    tc::split_tf32(w0t[e], hi, lo);
    const uint32_t off = tc::kmajor_offset(o, i, kC) / 4;
    sm.wb_hi[off] = hi;
    sm.wb_lo[off] = lo;
  }
  constexpr bool kHasBias = EPI == kEpiGelu || EPI == kEpiGeluSavePre;  // the adjoint epilogues take none
  if (tid < kC) sm.bias[tid] = (kHasBias && bias != nullptr) ? bias[tid] : 0.f;
  tc::fence_proxy_async_smem();   // the constant operands above are read by the tensor cores
  __syncthreads();
  pdl_wait();  // everything above touched only weights / the constant E table; z and x come from the chain
  pdl_launch_dependents();

  const int first = blockIdx.x * kBtWG + wg, stride = gridDim.x * kBtWG;
  float* ax_hi = sm.ax_hi[wg];
  float* ax_lo = sm.ax_lo[wg];
  float* bz_hi = sm.bz_hi[wg];
  float* bz_lo = sm.bz_lo[wg];
  BtRegs<TAct> regs;
  if (first < n_tiles) bt_prefetch<TAct>(regs, x, z, first, t);
  for (int tile = first; tile < n_tiles; tile += stride) {
    // this pipeline's operands were last read by the MMAs of its previous tile, which every thread waited for
    bt_split_store<TAct>(regs, ax_hi, ax_lo, bz_hi, bz_lo, sm.bias, t);
    tc::fence_proxy_async_smem();
    tc::named_barrier(1 + wg, 128);
    // prefetch AFTER the fence: the membar inside fence.proxy.async would otherwise wait for these loads
    if (tile + stride < n_tiles) bt_prefetch<TAct>(regs, x, z, tile + stride, t);
    float acc[16];
    tc::wg_fence();
    {
      // 3xTF32: pass 0 = hi*hi, pass 1 = lo*hi, pass 2 = hi*lo (A part, B part)
      const uint32_t a_e[3] = {tc::smem_addr(sm.e_hi), tc::smem_addr(sm.e_lo), tc::smem_addr(sm.e_hi)};
      const uint32_t b_z[3] = {tc::smem_addr(bz_hi), tc::smem_addr(bz_hi), tc::smem_addr(bz_lo)};
      const uint32_t a_x[3] = {tc::smem_addr(ax_hi), tc::smem_addr(ax_lo), tc::smem_addr(ax_hi)};
      const uint32_t b_w[3] = {tc::smem_addr(sm.wb_hi), tc::smem_addr(sm.wb_hi), tc::smem_addr(sm.wb_lo)};
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {
#pragma unroll
        for (int ks = 0; ks < kKE / 8; ++ks)
          tc::wg_tf32_ss_n32(acc, tc::make_smem_desc(a_e[pass] + ks * 2 * kLboA, kLboA, 128),
                             tc::make_smem_desc(b_z[pass] + ks * 2 * kLboB, kLboB, 128), (pass | ks) ? 1u : 0u);
        if (kBf16 && pass == 1) continue;  // conv-part A has no lo component
#pragma unroll
        for (int ks = 0; ks < kKConv / 8; ++ks)
          tc::wg_tf32_ss_n32(acc, tc::make_smem_desc(a_x[pass] + ks * 2 * kLboA, kLboA, 128),
                             tc::make_smem_desc(b_w[pass] + ks * 2 * kLboB, kLboB, 128), 1u);
      }
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_fence_acc(acc);
    // epilogue: acc[4 i + 2 hh + e] = D[px = 16 wq + lane/4 + 8 hh][o = 8 i + 2 (lane%4) + e]
    const int b = tile / kBtTilesPerSample, h = tile % kBtTilesPerSample;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int px = 16 * wq + (lane >> 2) + 8 * hh, o = 8 * i + 2 * (lane & 3);
        float2 p = make_float2(acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
        const size_t o0 = (static_cast<size_t>(b) * kC + o) * kHW + h * kW + px, o1 = o0 + kHW;
        if constexpr (EPI == kEpiGelu || EPI == kEpiGeluSavePre) {  // the accumulator already includes the bias
          if constexpr (EPI == kEpiGeluSavePre) {
            pre_out[o0] = p.x;
            pre_out[o1] = p.y;
          }
          p = gelu_erf2(p);
        } else if constexpr (EPI == kEpiMulDgelu) {
          p.x *= dgelu_erf(__ldg(pre_in + o0));
          p.y *= dgelu_erf(__ldg(pre_in + o1));
        }
        bt_store(out + o0, p.x);
        bt_store(out + o1, p.y);
      }
  }
}

// ------------------------------------------------------------------------------------------------
// Constant A-operand image of the C2R stage: rows m = w (one image row), columns k = 2 ky + ri;
// E = c_ky cos(2 pi ky w/64) (ri=0), -c_ky sin(2 pi ky w/64) (ri=1), c_0 = s0, c_ky = s1 otherwise.  The (ky=0, ri=1)
// column would be identically zero (C2R drops Im of the ky=0 column); it holds 1 instead and the matching B row holds
// the conv bias, which folds the bias add into the MMA.  Built in float64, split into tf32 hi/lo (round-to-nearest),
// laid out K-major: hi image then lo image.  Also the constant of block_fused_kernel (with s0 = 1/HW, s1 = 2/HW).
// ------------------------------------------------------------------------------------------------
void c2r_operand_table(float* host, double s0, double s1) {
  for (int i = 0; i < kETabFloats; ++i) host[i] = 0.f;
  for (int w = 0; w < kBtM; ++w)
    for (int ky = 0; ky < kM2; ++ky) {
      const double ang = 2.0 * 3.14159265358979323846 * ((ky * w) % 64) / 64.0;
      const double c = ky == 0 ? s0 : s1;
      const double val[2] = {c * cos(ang), ky == 0 ? 1.0 : -c * sin(ang)};  // ky = 0, ri = 1: the bias column
      for (int ri = 0; ri < 2; ++ri) {
        const float hi = tc::round_tf32(static_cast<float>(val[ri]));
        const float lo = tc::round_tf32(static_cast<float>(val[ri] - static_cast<double>(hi)));
        const uint32_t off = tc::kmajor_offset(w, 2 * ky + ri, kBtM) / 4;
        host[off] = hi;
        host[kBtM * kKE + off] = lo;
      }
    }
}

static float* g_etab[64] = {nullptr};

static cudaError_t ensure_etab(const float** out, cudaStream_t stream) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (g_etab[dev] == nullptr) {
    static float host[kETabFloats];
    c2r_operand_table(host, 1.0, 1.0);   // Z arrives scaled by inv_kx
    float* d = nullptr;
    e = cudaMalloc(&d, sizeof(host));
    if (e != cudaSuccess) return e;
    e = cudaMemcpyAsync(d, host, sizeof(host), cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(stream);  // `host` is static: make sure the copy has consumed it
    if (e != cudaSuccess) return e;
    g_etab[dev] = d;
  }
  *out = g_etab[dev];
  return cudaSuccess;
}

void block_tc_release(int dev) {
  if (dev >= 0 && dev < 64 && g_etab[dev] != nullptr) {
    cudaFree(g_etab[dev]);
    g_etab[dev] = nullptr;
  }
}

template <typename TAct, int EPI>
static cudaError_t launch_one(const void* z, const void* x, const float* w0t, const float* bias, void* out,
                              float* pre_out, const float* pre_in, int batch, cudaStream_t stream) {
  auto kern = block_tc_kernel<TAct, EPI>;
  constexpr size_t smem = sizeof(BtSmem);
  static PerDeviceLaunch pd;
  int n_sm = 0;
  cudaError_t e = per_device_setup(kern, smem, pd, &n_sm);
  if (e != cudaSuccess) return e;
  const float* etab = nullptr;
  e = ensure_etab(&etab, stream);
  if (e != cudaSuccess) return e;
  const int n_tiles = batch * kBtTilesPerSample;
  const int want = (n_tiles + kBtWG - 1) / kBtWG;
  const int grid = want < n_sm ? want : n_sm;
  return launch_chained(kern, dim3(grid), dim3(kBtThreads), smem, stream, static_cast<const float*>(z),
                        static_cast<const TAct*>(x), w0t, bias, etab, static_cast<TAct*>(out), pre_out, pre_in, n_tiles);
}

template <typename TAct>
cudaError_t launch_block_tc(int epi, const void* z, const void* x, const float* w0t, const float* bias, void* out,
                            float* pre_out, const float* pre_in, int batch, cudaStream_t stream) {
  switch (epi) {
    case kEpiGelu: return launch_one<TAct, kEpiGelu>(z, x, w0t, bias, out, pre_out, pre_in, batch, stream);
    case kEpiGeluSavePre: return launch_one<TAct, kEpiGeluSavePre>(z, x, w0t, bias, out, pre_out, pre_in, batch, stream);
    case kEpiMulDgelu: return launch_one<TAct, kEpiMulDgelu>(z, x, w0t, bias, out, pre_out, pre_in, batch, stream);
    case kEpiPlain: return launch_one<TAct, kEpiPlain>(z, x, w0t, bias, out, pre_out, pre_in, batch, stream);
    default: return cudaErrorInvalidValue;
  }
}

template cudaError_t launch_block_tc<float>(int, const void*, const void*, const float*, const float*, void*, float*,
                                            const float*, int, cudaStream_t);
template cudaError_t launch_block_tc<__nv_bfloat16>(int, const void*, const void*, const float*, const float*, void*,
                                                    float*, const float*, int, cudaStream_t);

}  // namespace fno
