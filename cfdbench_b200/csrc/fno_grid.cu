// Grid-generic fp32 kernels: the same network on any H x W frame with 24 <= H, W <= 128 (CFDBench's tube and dam
// problems feed 66 x 65 frames, reference src/utils/autoregressive.py:24-26).  The 64 x 64 kernels tile by one 64-pixel
// image row and move planes with 16-byte bulk copies; a 65-float row fits neither, so every per-pixel stage here tiles the
// FLATTENED pixel index of one sample and masks the tail, and every access to a caller's plane is a scalar load / store
// (a 66 x 65 plane is 17,160 B: every odd plane of a user tensor starts on an 8-byte, not a 16-byte, boundary).
//
// Layouts (all chosen so that the grid-independent kernels -- mode mix, spectral wgrad, unpack, reduce_partials -- are
// reused unchanged):
//   activations / pre / d   [B][32][H*W] float32, planes unpadded
//   modes (xm, ym, gm)      [288][B][32] complex64, mode k = kxi*12 + ky, kxi >= 12 <-> kx = H - 24 + kxi
//   z                       [B][H][24][32] float32: Z[b][h][2 ky + (re|im)][o]
//
// Kernels (all FFMA, fp32 end to end):
//   grid_lift_kernel        channel assembly + fc0, one thread per pixel
//   grid_dft_kernel         truncated forward rDFT of one plane per CTA: along w (12 ky) then along h (24 kx)
//   grid_inv_kx_kernel      inverse DFT along kx of the 24 kept rows, one CTA per sample, thread = (ky, o)
//   grid_block_out_kernel   C2R along w + w0 1x1 + bias + epilogue, one thread per pixel of a 128-pixel tile
//   grid_project_kernel     fc1 + GELU + fc2 + mask, one thread per pixel
//   grid_project_bwd_kernel dpre of the last block, dz1, and per-CTA partial rows of fc2.weight | fc1.bias | fc2.bias
//   grid_chan_outer_kernel  G[j][i] = sum P[b][j][p] Q[b][i][p] (+ bias column), per-CTA partial rows
//   grid_lift_bwd_kernel    fc0 weight / bias partial rows and the data adjoint into d_inputs / d_case_params
// Small gradients are written as per-CTA partial rows by a FIXED number of CTAs with a fixed tile order and summed in
// index order by reduce_partials: no float atomics, bit-reproducible gradients.
//
// Twiddles: per (device, H, W) one table [H + W] of (cos, sin)(2 pi m / n) evaluated in float64 on the host and stored as
// float32; fno_destroy releases it.
#include <math.h>
#include <mutex>
#include <vector>

#include "fno_common.cuh"

namespace fno {

cudaError_t launch_reduce_partials(const float*, int, int, float*, int, float*, int, float*, int, int, cudaStream_t);

constexpr int kGridMin = 24;
constexpr int kGridMax = 128;
constexpr int kZK2 = 2 * kM2;   // 24 real columns of a z row

// ------------------------------------------------------------------------------------------------ twiddle tables
namespace {
struct GridTable {
  int dev, h, w;
  float2* d;
};
std::mutex g_tab_mu;
std::vector<GridTable> g_tabs;
}  // namespace

// (cos, sin)(2 pi m / h) for m < h, then (cos, sin)(2 pi m / w) for m < w
static cudaError_t grid_tables(int h, int w, const float2** out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(g_tab_mu);
  for (const GridTable& t : g_tabs)
    if (t.dev == dev && t.h == h && t.w == w) {
      *out = t.d;
      return cudaSuccess;
    }
  std::vector<float2> host(h + w);
  const double two_pi = 6.283185307179586476925286766559;
  for (int m = 0; m < h; ++m)
    host[m] = make_float2(static_cast<float>(cos(two_pi * m / h)), static_cast<float>(sin(two_pi * m / h)));
  for (int m = 0; m < w; ++m)
    host[h + m] = make_float2(static_cast<float>(cos(two_pi * m / w)), static_cast<float>(sin(two_pi * m / w)));
  float2* d = nullptr;
  e = cudaMalloc(&d, host.size() * sizeof(float2));
  if (e != cudaSuccess) return e;
  e = cudaMemcpy(d, host.data(), host.size() * sizeof(float2), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d);
    return e;
  }
  g_tabs.push_back({dev, h, w, d});
  *out = d;
  return cudaSuccess;
}

void grid_tables_release(int dev) {
  std::lock_guard<std::mutex> lk(g_tab_mu);
  for (size_t i = 0; i < g_tabs.size();) {
    if (g_tabs[i].dev == dev) {
      cudaFree(g_tabs[i].d);
      g_tabs.erase(g_tabs.begin() + i);
    } else {
      ++i;
    }
  }
}

bool grid_ok(int h, int w) { return h >= kGridMin && h <= kGridMax && w >= kGridMin && w <= kGridMax; }

__device__ __forceinline__ int kx_of(int kxi, int h) { return kxi < kM1 ? kxi : h - kKX + kxi; }

// ------------------------------------------------------------------------------------------------ lift
constexpr int kGlThreads = 256;

__global__ void __launch_bounds__(kGlThreads)
    grid_lift_kernel(const float* __restrict__ inputs, const float* __restrict__ mask, const float* __restrict__ params,
                     const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gx,
                     const float* __restrict__ gy, float* __restrict__ out, int p, int h, int wd) {
  __shared__ float sw[kC][5];
  __shared__ float scb[kC];
  const int b = blockIdx.y, tid = threadIdx.x, nin = 5 + p, hw = h * wd;
  if (tid < kC) {
    float cb = bias[tid];
    for (int q = 0; q < p; ++q) cb = fmaf(w[tid * nin + 5 + q], params[b * p + q], cb);
    scb[tid] = cb;
#pragma unroll
    for (int q = 0; q < 5; ++q) sw[tid][q] = w[tid * nin + q];
  }
  __syncthreads();
  const int pix = blockIdx.x * kGlThreads + tid;
  if (pix >= hw) return;
  const int hh = pix / wd, ww = pix - hh * wd;
  const float u = inputs[(static_cast<size_t>(b) * 2 + 0) * hw + pix];
  const float v = inputs[(static_cast<size_t>(b) * 2 + 1) * hw + pix];
  const float m = mask[static_cast<size_t>(b) * hw + pix];
  const float xh = gx[hh], yw = gy[ww];
  float* dst = out + static_cast<size_t>(b) * kC * hw + pix;
#pragma unroll 8
  for (int c = 0; c < kC; ++c) {
    const float base = fmaf(sw[c][3], xh, scb[c]);
    dst[static_cast<size_t>(c) * hw] = fmaf(sw[c][0], u, fmaf(sw[c][1], v, fmaf(sw[c][2], m, fmaf(sw[c][4], yw, base))));
  }
}

cudaError_t launch_grid_lift(const float* inputs, const float* mask, const float* params, const float* w, const float* bias,
                             const float* gx, const float* gy, float* out, int batch, int p, int h, int wd,
                             cudaStream_t stream) {
  if (p < 0 || p > kMaxCaseParams) return cudaErrorInvalidValue;
  dim3 grid((h * wd + kGlThreads - 1) / kGlThreads, batch);
  grid_lift_kernel<<<grid, kGlThreads, 0, stream>>>(inputs, mask, params, w, bias, gx, gy, out, p, h, wd);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ forward rDFT
// One CTA per (sample, channel) plane.  Shared memory: F[w][ky] = e^{-2 pi i ky w / W}, G[h][kxi] = e^{-2 pi i kx h / H},
// T[h][ky] (the plane transformed along w), then the plane itself with an odd row pitch (conflict-free column walks).
constexpr int kGdThreads = 128;

static size_t grid_dft_smem(int h, int w) {
  return (static_cast<size_t>(w) * kM2 + static_cast<size_t>(h) * kKX + static_cast<size_t>(h) * kM2) * sizeof(float2) +
         static_cast<size_t>(h) * (w | 1) * sizeof(float);
}

__global__ void __launch_bounds__(kGdThreads)
    grid_dft_kernel(const float* __restrict__ x, float2* __restrict__ xm, const float2* __restrict__ tab, int h, int wd,
                    int batch, float s0, float s1) {
  extern __shared__ float4 g_dft_smem[];
  float2* F = reinterpret_cast<float2*>(g_dft_smem);
  float2* G = F + wd * kM2;
  float2* T = G + h * kKX;
  float* xs = reinterpret_cast<float*>(T + h * kM2);
  const int plane = blockIdx.x, tid = threadIdx.x, pitch = wd | 1;
  const float2* tw_h = tab;
  const float2* tw_w = tab + h;
  for (int i = tid; i < wd * kM2; i += kGdThreads) {
    const int w = i / kM2, ky = i - w * kM2;
    const float2 t = tw_w[(ky * w) % wd];
    F[i] = make_float2(t.x, -t.y);
  }
  for (int i = tid; i < h * kKX; i += kGdThreads) {
    const int hh = i / kKX, kxi = i - hh * kKX;
    const float2 t = tw_h[(kx_of(kxi, h) * hh) % h];
    G[i] = make_float2(t.x, -t.y);
  }
  const float* src = x + static_cast<size_t>(plane) * h * wd;
  for (int i = tid; i < h * wd; i += kGdThreads) {
    const int hh = i / wd;
    xs[hh * pitch + (i - hh * wd)] = src[i];
  }
  __syncthreads();
  // along w: item = (row, half of the 12 ky)
  for (int item = tid; item < 2 * h; item += kGdThreads) {
    const int hh = item >> 1, k0 = (item & 1) * (kM2 / 2);
    float re[kM2 / 2], im[kM2 / 2];
#pragma unroll
    for (int k = 0; k < kM2 / 2; ++k) re[k] = im[k] = 0.f;
    const float* row = xs + hh * pitch;
    for (int w = 0; w < wd; ++w) {
      const float xv = row[w];
      const float4* f = reinterpret_cast<const float4*>(F + w * kM2 + k0);   // 6 twiddles = 3 x 16 B
#pragma unroll
      for (int k = 0; k < kM2 / 4; ++k) {
        const float4 t = f[k];
        re[2 * k] = fmaf(xv, t.x, re[2 * k]);
        im[2 * k] = fmaf(xv, t.y, im[2 * k]);
        re[2 * k + 1] = fmaf(xv, t.z, re[2 * k + 1]);
        im[2 * k + 1] = fmaf(xv, t.w, im[2 * k + 1]);
      }
    }
#pragma unroll
    for (int k = 0; k < kM2 / 2; ++k) T[hh * kM2 + k0 + k] = make_float2(re[k], im[k]);
  }
  __syncthreads();
  // along h: item = mode k = kxi * 12 + ky
  for (int k = tid; k < kModes; k += kGdThreads) {
    const int kxi = k / kM2, ky = k - kxi * kM2;
    float re = 0.f, im = 0.f;
    for (int hh = 0; hh < h; ++hh) {
      const float2 t = T[hh * kM2 + ky], g = G[hh * kKX + kxi];
      re = fmaf(t.x, g.x, fmaf(-t.y, g.y, re));
      im = fmaf(t.x, g.y, fmaf(t.y, g.x, im));
    }
    const float s = ky == 0 ? s0 : s1;
    xm[static_cast<size_t>(k) * batch * kC + plane] = make_float2(re * s, im * s);
  }
}

cudaError_t launch_grid_dft(const float* x, void* xm, int batch, int h, int wd, float s0, float s1, cudaStream_t stream) {
  static PerDeviceLaunch st;
  cudaError_t e = per_device_setup(grid_dft_kernel, grid_dft_smem(kGridMax, kGridMax), st);
  if (e != cudaSuccess) return e;
  const float2* tab = nullptr;
  if ((e = grid_tables(h, wd, &tab)) != cudaSuccess) return e;
  grid_dft_kernel<<<batch * kC, kGdThreads, grid_dft_smem(h, wd), stream>>>(x, static_cast<float2*>(xm), tab, h, wd, batch,
                                                                           s0, s1);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ inverse along kx
constexpr int kGiThreads = kM2 * kC;   // 384: thread = (ky, o), one CTA per sample

__global__ void __launch_bounds__(kGiThreads)
    grid_inv_kx_kernel(const float2* __restrict__ ym, float* __restrict__ z, const float2* __restrict__ tab, int h,
                       float s0, float s1) {
  extern __shared__ float2 g_ik_tab[];   // [h][24]: e^{+2 pi i kx h / H}
  const int b = blockIdx.x, batch = gridDim.x, tid = threadIdx.x;
  for (int i = tid; i < h * kKX; i += kGiThreads) {
    const int hh = i / kKX, kxi = i - hh * kKX;
    g_ik_tab[i] = tab[(kx_of(kxi, h) * hh) % h];
  }
  const int ky = tid >> 5, o = tid & 31;
  float yre[kKX], yim[kKX];
#pragma unroll
  for (int kxi = 0; kxi < kKX; ++kxi) {
    const float2 v = ym[(static_cast<size_t>(kxi * kM2 + ky) * batch + b) * kC + o];
    yre[kxi] = v.x;
    yim[kxi] = v.y;
  }
  __syncthreads();
  const float s = ky == 0 ? s0 : s1;
  float* zb = z + (static_cast<size_t>(b) * h * kZK2 + 2 * ky) * kC + o;
  for (int hh = 0; hh < h; ++hh) {
    float re = 0.f, im = 0.f;
#pragma unroll
    for (int kxi = 0; kxi < kKX; ++kxi) {
      const float2 g = g_ik_tab[hh * kKX + kxi];
      re = fmaf(yre[kxi], g.x, fmaf(-yim[kxi], g.y, re));
      im = fmaf(yre[kxi], g.y, fmaf(yim[kxi], g.x, im));
    }
    zb[static_cast<size_t>(hh) * kZK2 * kC] = re * s;
    zb[static_cast<size_t>(hh) * kZK2 * kC + kC] = im * s;
  }
}

cudaError_t launch_grid_inv_kx(const void* ym, float* z, int batch, int h, int wd, float s0, float s1, cudaStream_t stream) {
  const float2* tab = nullptr;
  cudaError_t e = grid_tables(h, wd, &tab);
  if (e != cudaSuccess) return e;
  grid_inv_kx_kernel<<<batch, kGiThreads, static_cast<size_t>(h) * kKX * sizeof(float2), stream>>>(
      static_cast<const float2*>(ym), z, tab, h, s0, s1);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ block output
// out[b][o][p] = epi( sum_ky Re(Z[b][h][ky][o] e^{2 pi i ky w / W}) + sum_i W[i][o] x[b][i][p] + bias[o] ), p = h W + w.
// A 128-pixel tile of the flattened index touches at most 7 image rows when W >= 24; their z rows are staged in shared
// memory.  Epilogues as fno_block_out: GELU, GELU_SAVE_PRE (also stores the pre-activation), MUL_DGELU (multiplies by
// GELU'(pre_in)), PLAIN.
constexpr int kGbThreads = 128;
constexpr int kGbRows = (kGbThreads - 1) / kGridMin + 2;   // 7

template <int EPI>
__global__ void __launch_bounds__(kGbThreads)
    grid_block_out_kernel(const float* __restrict__ z, const float* __restrict__ x, const float* __restrict__ wt,
                          const float* __restrict__ bias, float* __restrict__ out, float* __restrict__ pre_out,
                          const float* __restrict__ pre_in, const float2* __restrict__ tab, int h, int wd) {
  __shared__ __align__(16) float zs[kGbRows][kZK2][kC];
  __shared__ __align__(16) float ws[kC][kC];
  __shared__ float bs[kC];
  __shared__ float2 tw[kGridMax];
  const int b = blockIdx.y, tid = threadIdx.x, hw = h * wd;
  const int p0 = blockIdx.x * kGbThreads;
  const int r0 = p0 / wd;
  const int r1 = min(h - 1, (p0 + kGbThreads - 1) / wd);
  {
    const float4* zsrc = reinterpret_cast<const float4*>(z + (static_cast<size_t>(b) * h + r0) * kZK2 * kC);
    float4* zdst = reinterpret_cast<float4*>(&zs[0][0][0]);
    for (int i = tid; i < (r1 - r0 + 1) * kZK2 * kC / 4; i += kGbThreads) zdst[i] = zsrc[i];
  }
  for (int i = tid; i < kC * kC; i += kGbThreads) (&ws[0][0])[i] = wt[i];
  if (tid < kC) bs[tid] = bias ? bias[tid] : 0.f;
  for (int i = tid; i < wd; i += kGbThreads) tw[i] = tab[h + i];
  __syncthreads();
  const int pix = p0 + tid;
  if (pix >= hw) return;
  const int hh = pix / wd, ww = pix - hh * wd;
  const float* zr = &zs[hh - r0][0][0];
  float acc[kC];
#pragma unroll
  for (int o = 0; o < kC; ++o) acc[o] = bs[o];
  int idx = 0;   // ky * ww mod W
#pragma unroll 2
  for (int ky = 0; ky < kM2; ++ky) {
    const float2 t = tw[idx];
    idx += ww;
    if (idx >= wd) idx -= wd;
    const float4* zre = reinterpret_cast<const float4*>(zr + (2 * ky) * kC);
    const float4* zim = reinterpret_cast<const float4*>(zr + (2 * ky + 1) * kC);
#pragma unroll
    for (int o4 = 0; o4 < kC / 4; ++o4) {
      const float4 re = zre[o4], im = zim[o4];
      acc[4 * o4 + 0] = fmaf(re.x, t.x, fmaf(-im.x, t.y, acc[4 * o4 + 0]));
      acc[4 * o4 + 1] = fmaf(re.y, t.x, fmaf(-im.y, t.y, acc[4 * o4 + 1]));
      acc[4 * o4 + 2] = fmaf(re.z, t.x, fmaf(-im.z, t.y, acc[4 * o4 + 2]));
      acc[4 * o4 + 3] = fmaf(re.w, t.x, fmaf(-im.w, t.y, acc[4 * o4 + 3]));
    }
  }
  const float* xb = x + static_cast<size_t>(b) * kC * hw + pix;
#pragma unroll 4
  for (int i = 0; i < kC; ++i) {
    const float xv = xb[static_cast<size_t>(i) * hw];
    const float4* wr = reinterpret_cast<const float4*>(&ws[i][0]);
#pragma unroll
    for (int o4 = 0; o4 < kC / 4; ++o4) {
      const float4 wv = wr[o4];
      acc[4 * o4 + 0] = fmaf(wv.x, xv, acc[4 * o4 + 0]);
      acc[4 * o4 + 1] = fmaf(wv.y, xv, acc[4 * o4 + 1]);
      acc[4 * o4 + 2] = fmaf(wv.z, xv, acc[4 * o4 + 2]);
      acc[4 * o4 + 3] = fmaf(wv.w, xv, acc[4 * o4 + 3]);
    }
  }
  const size_t base = static_cast<size_t>(b) * kC * hw + pix;
#pragma unroll
  for (int o = 0; o < kC; ++o) {
    const size_t off = base + static_cast<size_t>(o) * hw;
    const float v = acc[o];
    if constexpr (EPI == 0) {
      out[off] = gelu_erf(v);
    } else if constexpr (EPI == 1) {
      pre_out[off] = v;
      out[off] = gelu_erf(v);
    } else if constexpr (EPI == 2) {
      out[off] = v * dgelu_erf(pre_in[off]);
    } else {
      out[off] = v;
    }
  }
}

cudaError_t launch_grid_block_out(int epi, const float* z, const float* x, const float* wt, const float* bias, float* out,
                                  float* pre_out, const float* pre_in, int batch, int h, int wd, cudaStream_t stream) {
  const float2* tab = nullptr;
  cudaError_t e = grid_tables(h, wd, &tab);
  if (e != cudaSuccess) return e;
  dim3 grid((h * wd + kGbThreads - 1) / kGbThreads, batch);
  switch (epi) {
    case 0: grid_block_out_kernel<0><<<grid, kGbThreads, 0, stream>>>(z, x, wt, bias, out, pre_out, pre_in, tab, h, wd); break;
    case 1: grid_block_out_kernel<1><<<grid, kGbThreads, 0, stream>>>(z, x, wt, bias, out, pre_out, pre_in, tab, h, wd); break;
    case 2: grid_block_out_kernel<2><<<grid, kGbThreads, 0, stream>>>(z, x, wt, bias, out, pre_out, pre_in, tab, h, wd); break;
    case 3: grid_block_out_kernel<3><<<grid, kGbThreads, 0, stream>>>(z, x, wt, bias, out, pre_out, pre_in, tab, h, wd); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ projection
constexpr int kGpThreads = 128;

__global__ void __launch_bounds__(kGpThreads)
    grid_project_kernel(const float* __restrict__ a, const float* __restrict__ w1, const float* __restrict__ b1,
                        const float* __restrict__ w2, const float* __restrict__ b2, const float* __restrict__ mask,
                        float* __restrict__ preds, int hw) {
  __shared__ __align__(16) float w1s[kProj][kC];
  __shared__ float b1s[kProj];
  __shared__ float w2s[2][kProj];
  const int b = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < kProj * kC; i += kGpThreads) (&w1s[0][0])[i] = w1[i];
  for (int i = tid; i < kProj; i += kGpThreads) {
    b1s[i] = b1[i];
    w2s[0][i] = w2[i];
    w2s[1][i] = w2[kProj + i];
  }
  __syncthreads();
  const int pix = blockIdx.x * kGpThreads + tid;
  if (pix >= hw) return;
  float av[kC];
  const float* ab = a + static_cast<size_t>(b) * kC * hw + pix;
#pragma unroll
  for (int i = 0; i < kC; ++i) av[i] = ab[static_cast<size_t>(i) * hw];
  float o0 = 0.f, o1 = 0.f;
#pragma unroll 2
  for (int j = 0; j < kProj; ++j) {
    float zv = b1s[j];
    const float4* wr = reinterpret_cast<const float4*>(&w1s[j][0]);
#pragma unroll
    for (int i4 = 0; i4 < kC / 4; ++i4) {
      const float4 wv = wr[i4];
      zv = fmaf(wv.x, av[4 * i4 + 0], zv);
      zv = fmaf(wv.y, av[4 * i4 + 1], zv);
      zv = fmaf(wv.z, av[4 * i4 + 2], zv);
      zv = fmaf(wv.w, av[4 * i4 + 3], zv);
    }
    const float g = gelu_erf(zv);
    o0 = fmaf(w2s[0][j], g, o0);
    o1 = fmaf(w2s[1][j], g, o1);
  }
  const float m = mask[static_cast<size_t>(b) * hw + pix];
  preds[(static_cast<size_t>(b) * 2 + 0) * hw + pix] = (o0 + b2[0]) * m;
  preds[(static_cast<size_t>(b) * 2 + 1) * hw + pix] = (o1 + b2[1]) * m;
}

cudaError_t launch_grid_project(const float* a, const float* w1, const float* b1, const float* w2, const float* b2,
                                const float* mask, float* preds, int batch, int hw, cudaStream_t stream) {
  dim3 grid((hw + kGpThreads - 1) / kGpThreads, batch);
  grid_project_kernel<<<grid, kGpThreads, 0, stream>>>(a, w1, b1, w2, b2, mask, preds, hw);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ projection backward
// A fixed number of CTAs walk 32-pixel tiles (sample-major) in a fixed order.  Per tile:
//   phase A, thread = fc1 channel j: z1 = fc1(a) recomputed, dz1[j][p] = (w2[:, j] . dout[p]) GELU'(z1) into shared
//            memory, and the running sums of fc2.weight (dout GELU(z1)) and fc1.bias (dz1) in registers;
//   phase B, thread = (pixel, 8 channels i): da[i] = sum_j w1[j][i] dz1[j][p], dpre = da GELU'(pre); dz1 is stored.
// dout = dpreds * mask.  Partial row: fc2.weight (2 x 128) | fc1.bias (128) | fc2.bias (2).
constexpr int kGqThreads = kProj;   // 128
constexpr int kGqPix = 32;
constexpr int kGqParts = 1024;
constexpr int kGqRow = 3 * kProj + 2;

__global__ void __launch_bounds__(kGqThreads)
    grid_project_bwd_kernel(const float* __restrict__ a, const float* __restrict__ dpreds, const float* __restrict__ mask,
                            const float* __restrict__ pre, const float* __restrict__ w1, const float* __restrict__ b1,
                            const float* __restrict__ w2, float* __restrict__ dpre_out, float* __restrict__ dz1,
                            float* __restrict__ partial, int nb, int hw) {
  __shared__ __align__(16) float w1s[kProj][kC];
  __shared__ __align__(16) float as[kC][kGqPix];
  __shared__ float dzs[kProj][kGqPix + 1];
  __shared__ float dout[2][kGqPix];
  const int tid = threadIdx.x;
  for (int i = tid; i < kProj * kC; i += kGqThreads) (&w1s[0][0])[i] = w1[i];
  const int j = tid;
  float wrow[kC];
#pragma unroll
  for (int i = 0; i < kC; ++i) wrow[i] = w1[j * kC + i];
  const float b1j = b1[j], w20 = w2[j], w21 = w2[kProj + j];
  float acc_w20 = 0.f, acc_w21 = 0.f, acc_b1 = 0.f, acc_b2 = 0.f;
  const int tiles_per_sample = (hw + kGqPix - 1) / kGqPix;
  const int n_tiles = nb * tiles_per_sample;
  const int pp = tid & (kGqPix - 1), q = tid / kGqPix;   // phase B: pixel, channel group of 8
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int b = t / tiles_per_sample;
    const int p0 = (t - b * tiles_per_sample) * kGqPix;
    __syncthreads();   // the previous tile's phase B is done with as / dzs
    for (int i = tid; i < kC * kGqPix; i += kGqThreads) {
      const int c = i / kGqPix, p = i - c * kGqPix;
      as[c][p] = p0 + p < hw ? a[(static_cast<size_t>(b) * kC + c) * hw + p0 + p] : 0.f;
    }
    if (tid < 2 * kGqPix) {
      const int c = tid / kGqPix, p = tid - c * kGqPix;
      dout[c][p] = p0 + p < hw ? dpreds[(static_cast<size_t>(b) * 2 + c) * hw + p0 + p] * mask[static_cast<size_t>(b) * hw + p0 + p]
                               : 0.f;
    }
    __syncthreads();
    if (tid < 2) {
      float s = 0.f;
      for (int p = 0; p < kGqPix; ++p) s += dout[tid][p];
      acc_b2 += s;
    }
    for (int p4 = 0; p4 < kGqPix; p4 += 4) {   // 4 pixels per pass: one 16-byte load feeds 4 FMAs
      float zv[4] = {b1j, b1j, b1j, b1j};
#pragma unroll
      for (int i = 0; i < kC; ++i) {
        const float4 av = *reinterpret_cast<const float4*>(&as[i][p4]);
        zv[0] = fmaf(wrow[i], av.x, zv[0]);
        zv[1] = fmaf(wrow[i], av.y, zv[1]);
        zv[2] = fmaf(wrow[i], av.z, zv[2]);
        zv[3] = fmaf(wrow[i], av.w, zv[3]);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int p = p4 + k;
        const float x = zv[k];
        const float ax = fabsf(x);
        const float e = 0.5f * erfc_abs_scaled(ax);
        const float g = fmaxf(x, 0.f) - ax * e;
        const float cdf = x >= 0.f ? 1.f - e : e;
        const float pdf = 0.3989422804014327f * ex2_approx(-0.7213475204444817f * x * x);
        const float dg = fmaf(x, pdf, cdf);
        const float d0 = dout[0][p], d1 = dout[1][p];
        const float dz = fmaf(w20, d0, w21 * d1) * dg;
        dzs[j][p] = dz;
        acc_w20 = fmaf(d0, g, acc_w20);
        acc_w21 = fmaf(d1, g, acc_w21);
        acc_b1 += dz;
      }
    }
    __syncthreads();
    const int pix = p0 + pp;
    float da[kC / 4];
#pragma unroll
    for (int k = 0; k < kC / 4; ++k) da[k] = 0.f;
#pragma unroll 4
    for (int jj = 0; jj < kProj; ++jj) {
      const float dz = dzs[jj][pp];
      const float4 wa = *reinterpret_cast<const float4*>(&w1s[jj][q * 8]);
      const float4 wb = *reinterpret_cast<const float4*>(&w1s[jj][q * 8 + 4]);
      da[0] = fmaf(wa.x, dz, da[0]);
      da[1] = fmaf(wa.y, dz, da[1]);
      da[2] = fmaf(wa.z, dz, da[2]);
      da[3] = fmaf(wa.w, dz, da[3]);
      da[4] = fmaf(wb.x, dz, da[4]);
      da[5] = fmaf(wb.y, dz, da[5]);
      da[6] = fmaf(wb.z, dz, da[6]);
      da[7] = fmaf(wb.w, dz, da[7]);
    }
    if (pix < hw) {
#pragma unroll
      for (int k = 0; k < kC / 4; ++k) {
        const size_t off = (static_cast<size_t>(b) * kC + q * 8 + k) * hw + pix;
        dpre_out[off] = da[k] * dgelu_erf(pre[off]);
      }
      for (int jj = q * (kProj / 4); jj < (q + 1) * (kProj / 4); ++jj)
        dz1[(static_cast<size_t>(b) * kProj + jj) * hw + pix] = dzs[jj][pp];
    }
  }
  if (partial) {
    float* row = partial + static_cast<size_t>(blockIdx.x) * kGqRow;
    row[j] = acc_w20;
    row[kProj + j] = acc_w21;
    row[2 * kProj + j] = acc_b1;
    if (tid < 2) row[3 * kProj + tid] = acc_b2;
  }
}

int grid_project_bwd_parts(int nb, int hw) {
  const int tiles = nb * ((hw + kGqPix - 1) / kGqPix);
  return tiles < kGqParts ? tiles : kGqParts;
}
int grid_project_bwd_row() { return kGqRow; }

cudaError_t launch_grid_project_bwd(const float* a, const float* dpreds, const float* mask, const float* pre, const float* w1,
                                    const float* b1, const float* w2, float* dpre_out, float* dz1, float* partial, int nb,
                                    int hw, cudaStream_t stream) {
  grid_project_bwd_kernel<<<grid_project_bwd_parts(nb, hw), kGqThreads, 0, stream>>>(a, dpreds, mask, pre, w1, b1, w2,
                                                                                     dpre_out, dz1, partial, nb, hw);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ channel outer products
// G[j][i] = sum_{b,p} P[b][j][p] Q[b][i][p] and bias[j] = sum_{b,p} P[b][j][p] over nb samples of hw pixels.  A fixed
// number of CTAs walk 32-pixel tiles in a fixed order; thread (tj, ti) owns an RJ x RI block.  Partial row: G (NJ x NI,
// row-major) | bias (NJ).
constexpr int kGcThreads = 256;
constexpr int kGcPix = 32;
constexpr int kGcParts = 528;

template <int NJ, int NI>
__global__ void __launch_bounds__(kGcThreads)
    grid_chan_outer_kernel(const float* __restrict__ P, const float* __restrict__ Q, float* __restrict__ partial, int nb,
                           int hw) {
  constexpr int RI = 4;
  constexpr int TI = NI / RI;                        // 8
  constexpr int TJ = kGcThreads / TI;                // 32
  constexpr int RJ = NJ / TJ;                        // 4 (NJ = 128) or 1 (NJ = 32)
  constexpr int PJ = NJ + 4, PI = NI + 4;
  __shared__ __align__(16) float ps[kGcPix][PJ];
  __shared__ __align__(16) float qs[kGcPix][PI];
  const int tid = threadIdx.x, ti = tid % TI, tj = tid / TI;
  float acc[RJ][RI], bacc[RJ];
#pragma unroll
  for (int a = 0; a < RJ; ++a) {
    bacc[a] = 0.f;
#pragma unroll
    for (int c = 0; c < RI; ++c) acc[a][c] = 0.f;
  }
  const int tiles_per_sample = (hw + kGcPix - 1) / kGcPix;
  const int n_tiles = nb * tiles_per_sample;
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int b = t / tiles_per_sample;
    const int p0 = (t - b * tiles_per_sample) * kGcPix;
    __syncthreads();
    for (int i = tid; i < NJ * kGcPix; i += kGcThreads) {
      const int jj = i / kGcPix, p = i - jj * kGcPix;
      ps[p][jj] = p0 + p < hw ? P[(static_cast<size_t>(b) * NJ + jj) * hw + p0 + p] : 0.f;
    }
    for (int i = tid; i < NI * kGcPix; i += kGcThreads) {
      const int ii = i / kGcPix, p = i - ii * kGcPix;
      qs[p][ii] = p0 + p < hw ? Q[(static_cast<size_t>(b) * NI + ii) * hw + p0 + p] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int p = 0; p < kGcPix; ++p) {
      const float4 qv = *reinterpret_cast<const float4*>(&qs[p][ti * RI]);
      float pv[RJ];
      if constexpr (RJ == 4) {
        const float4 v = *reinterpret_cast<const float4*>(&ps[p][tj * RJ]);
        pv[0] = v.x; pv[1] = v.y; pv[2] = v.z; pv[3] = v.w;
      } else {
#pragma unroll
        for (int a = 0; a < RJ; ++a) pv[a] = ps[p][tj * RJ + a];
      }
#pragma unroll
      for (int a = 0; a < RJ; ++a) {
        acc[a][0] = fmaf(pv[a], qv.x, acc[a][0]);
        acc[a][1] = fmaf(pv[a], qv.y, acc[a][1]);
        acc[a][2] = fmaf(pv[a], qv.z, acc[a][2]);
        acc[a][3] = fmaf(pv[a], qv.w, acc[a][3]);
        bacc[a] += pv[a];
      }
    }
  }
  float* row = partial + static_cast<size_t>(blockIdx.x) * (NJ * NI + NJ);
#pragma unroll
  for (int a = 0; a < RJ; ++a) {
#pragma unroll
    for (int c = 0; c < RI; ++c) row[(tj * RJ + a) * NI + ti * RI + c] = acc[a][c];
    if (ti == 0) row[NJ * NI + tj * RJ + a] = bacc[a];
  }
}

int grid_chan_outer_parts(int nb, int hw) {
  const int tiles = nb * ((hw + kGcPix - 1) / kGcPix);
  return tiles < kGcParts ? tiles : kGcParts;
}

template <int NJ, int NI>
cudaError_t launch_grid_chan_outer(const float* P, const float* Q, float* partial, int* n_parts, int nb, int hw,
                                   cudaStream_t stream) {
  *n_parts = grid_chan_outer_parts(nb, hw);
  grid_chan_outer_kernel<NJ, NI><<<*n_parts, kGcThreads, 0, stream>>>(P, Q, partial, nb, hw);
  return cudaGetLastError();
}
template cudaError_t launch_grid_chan_outer<kProj, kC>(const float*, const float*, float*, int*, int, int, cudaStream_t);
template cudaError_t launch_grid_chan_outer<kC, kC>(const float*, const float*, float*, int*, int, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------ lift backward
// A fixed number of CTAs walk the samples in a fixed order.  Per sample: warp w forms, for channels j = w, w+8, .., the
// plane sums of dL/da0 times (u, v, mask, x, y, 1) (fixed-order warp reductions); the fc0 weight partials add those sums
// -- the case-parameter columns as param * sum(dL/da0) -- to the CTA's running row in shared memory; d_case_params[b][q] =
// sum_j fc0_w[j][5+q] sum(dL/da0[j]); d_inputs[b][c][p] = sum_j fc0_w[j][c] dL/da0[b][j][p].
// Partial row: fc0.weight (32 x (5+p)) | fc0.bias (32), stride kGlbRow.
// kHandOff (the rollout backward's sweep): d_inputs = (sum_j fc0_w[j][c] dL/da0) + add, `add` (or null) being the upstream
// gradient of the previous step's prediction, and d_case_params += instead of =.  `gate` (or null; kHandOff only, teacher
// forcing): where gate[b] != 0, d_inputs = add, a copy bit for bit; d_case_params and the partials still take b's share.
constexpr int kGlbThreads = 256;
constexpr int kGlbParts = 264;
constexpr int kGlbRow = kC * (5 + kMaxCaseParams) + kC;

template <bool kHandOff>
__global__ void __launch_bounds__(kGlbThreads)
    grid_lift_bwd_kernel(const float* __restrict__ da0, const float* __restrict__ inputs, const float* __restrict__ mask,
                         const float* __restrict__ params, const float* __restrict__ gx, const float* __restrict__ gy,
                         const float* __restrict__ fc0_w, float* __restrict__ partial, float* __restrict__ d_inputs,
                         float* __restrict__ d_params, const float* __restrict__ add,
                         const unsigned char* __restrict__ gate, int batch, int p, int h, int wd) {
  __shared__ float sums[kC][6];
  __shared__ float accw[kC * (5 + kMaxCaseParams)];
  __shared__ float accb[kC];
  __shared__ float wuv[2][kC];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nin = 5 + p, hw = h * wd;
  for (int i = tid; i < kC * nin; i += kGlbThreads) accw[i] = 0.f;
  if (tid < kC) {
    accb[tid] = 0.f;
    wuv[0][tid] = fc0_w[tid * nin + 0];
    wuv[1][tid] = fc0_w[tid * nin + 1];
  }
  const bool sums_needed = partial != nullptr || (d_params != nullptr && p > 0);
  for (int b = blockIdx.x; b < batch; b += gridDim.x) {
    __syncthreads();
    const float* db = da0 + static_cast<size_t>(b) * kC * hw;
    if (sums_needed) {
      constexpr int kJPerWarp = kC / (kGlbThreads / 32);   // 4
      float s[kJPerWarp][6];
#pragma unroll
      for (int k = 0; k < kJPerWarp; ++k)
#pragma unroll
        for (int f = 0; f < 6; ++f) s[k][f] = 0.f;
      for (int pix = lane; pix < hw; pix += 32) {
        const int hh = pix / wd, ww = pix - hh * wd;
        const float u = inputs[(static_cast<size_t>(b) * 2 + 0) * hw + pix];
        const float v = inputs[(static_cast<size_t>(b) * 2 + 1) * hw + pix];
        const float m = mask[static_cast<size_t>(b) * hw + pix];
        const float xh = gx[hh], yw = gy[ww];
#pragma unroll
        for (int k = 0; k < kJPerWarp; ++k) {
          const float d = db[static_cast<size_t>(warp + 8 * k) * hw + pix];
          s[k][0] = fmaf(d, u, s[k][0]);
          s[k][1] = fmaf(d, v, s[k][1]);
          s[k][2] = fmaf(d, m, s[k][2]);
          s[k][3] = fmaf(d, xh, s[k][3]);
          s[k][4] = fmaf(d, yw, s[k][4]);
          s[k][5] += d;
        }
      }
#pragma unroll
      for (int k = 0; k < kJPerWarp; ++k)
#pragma unroll
        for (int f = 0; f < 6; ++f) {
          float v = s[k][f];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0) sums[warp + 8 * k][f] = v;
        }
      __syncthreads();
      if (partial) {
        for (int i = tid; i < kC * nin; i += kGlbThreads) {
          const int jj = i / nin, f = i - jj * nin;
          accw[i] += f < 5 ? sums[jj][f] : sums[jj][5] * params[b * p + f - 5];
        }
        if (tid < kC) accb[tid] += sums[tid][5];
      }
      if (d_params && tid < p) {
        float d = 0.f;
        for (int jj = 0; jj < kC; ++jj) d = fmaf(fc0_w[jj * nin + 5 + tid], sums[jj][5], d);
        if constexpr (kHandOff) d_params[b * p + tid] += d;
        else d_params[b * p + tid] = d;
      }
    } else {
      __syncthreads();   // wuv visible
    }
    if (d_inputs) {
      const float* add_b = add != nullptr ? add + static_cast<size_t>(b) * 2 * hw : nullptr;
      if (kHandOff && add_b != nullptr && gate != nullptr && gate[b] != 0) {   // a forced sample: the carry is add alone
        for (int pix = tid; pix < hw; pix += kGlbThreads) {
          d_inputs[(static_cast<size_t>(b) * 2 + 0) * hw + pix] = add_b[pix];
          d_inputs[(static_cast<size_t>(b) * 2 + 1) * hw + pix] = add_b[hw + pix];
        }
        continue;
      }
      for (int pix = tid; pix < hw; pix += kGlbThreads) {
        float du = 0.f, dv = 0.f;
#pragma unroll 8
        for (int jj = 0; jj < kC; ++jj) {
          const float d = db[static_cast<size_t>(jj) * hw + pix];
          du = fmaf(wuv[0][jj], d, du);
          dv = fmaf(wuv[1][jj], d, dv);
        }
        if constexpr (kHandOff) {
          if (add_b != nullptr) {
            du += add_b[pix];
            dv += add_b[hw + pix];
          }
        }
        d_inputs[(static_cast<size_t>(b) * 2 + 0) * hw + pix] = du;
        d_inputs[(static_cast<size_t>(b) * 2 + 1) * hw + pix] = dv;
      }
    }
  }
  if (partial) {
    __syncthreads();
    float* row = partial + static_cast<size_t>(blockIdx.x) * kGlbRow;
    for (int i = tid; i < kC * nin; i += kGlbThreads) row[i] = accw[i];
    if (tid < kC) row[kC * nin + tid] = accb[tid];
  }
}

int grid_lift_bwd_parts(int batch) { return batch < kGlbParts ? batch : kGlbParts; }
int grid_lift_bwd_row() { return kGlbRow; }

// hand_off = 0: the single-step backward (`add` must be null); 1: the rollout sweep's mode described above the kernel
cudaError_t launch_grid_lift_bwd(const float* da0, const float* inputs, const float* mask, const float* params,
                                 const float* gx, const float* gy, const float* fc0_w, float* partial, float* d_inputs,
                                 float* d_params, const float* add, int hand_off, int batch, int p, int h, int wd,
                                 cudaStream_t stream, const unsigned char* gate) {
  if (p < 0 || p > kMaxCaseParams) return cudaErrorInvalidValue;
  if (hand_off)
    grid_lift_bwd_kernel<true><<<grid_lift_bwd_parts(batch), kGlbThreads, 0, stream>>>(
        da0, inputs, mask, params, gx, gy, fc0_w, partial, d_inputs, d_params, add, gate, batch, p, h, wd);
  else
    grid_lift_bwd_kernel<false><<<grid_lift_bwd_parts(batch), kGlbThreads, 0, stream>>>(
        da0, inputs, mask, params, gx, gy, fc0_w, partial, d_inputs, d_params, nullptr, nullptr, batch, p, h, wd);
  return cudaGetLastError();
}

// bytes of the partial-row scratch of the grid backward: project_bwd | chan_outer | lift_bwd regions
size_t grid_bwd_partials_floats() {
  return static_cast<size_t>(kGqParts) * kGqRow + static_cast<size_t>(kGcParts) * (kProj * kC + kProj) +
         static_cast<size_t>(kGlbParts) * kGlbRow;
}
size_t grid_partials_offset_co() { return static_cast<size_t>(kGqParts) * kGqRow; }
size_t grid_partials_offset_lb() { return grid_partials_offset_co() + static_cast<size_t>(kGcParts) * (kProj * kC + kProj); }

}  // namespace fno
