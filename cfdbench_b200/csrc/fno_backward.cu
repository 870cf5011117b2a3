// Backward-only kernels of the FNO training step (what torch.autograd derives for the reference's
// Fno2d.forward when train_auto.py:255 calls loss["nmse"].backward()).  The data-gradient path of a
// Fourier block reuses the forward kernels (K1 with the c_ky/4096 output scale, K2 with the
// conj-transposed weight pack, K3 with W0 un-transposed and the MUL_DGELU / PLAIN epilogues); this
// file holds what is new in the backward direction besides the project stage's (fno_project_bwd_tc.cu):
//   chan_outer_kernel    G[j][i] += sum_{b,pix} P[b][j][pix] Q[b][i][pix]  (1x1-conv weight gradients)
//   spectral_wgrad_kernel  gWk[k][i][o] = sum_b conj(X[b][k][i]) G[b][k][o]   (SURVEY.md 8a)
//   lift_bwd_kernel      gradients of fc0 (spatial feature columns + folded per-sample constants)
//   lift_bwd_data_kernel gradients w.r.t. the input frame (u, v) and the case parameters
#include "fno_common.cuh"

namespace fno {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// out[i] += sum over parts of partial[part][i] in a FIXED order: the second, deterministic half of every small-gradient
// reduction (the first half = one plain store per CTA).  Replaces float atomics, whose summation order -- and therefore the
// last bits of every gradient and the whole training trajectory -- changed from run to run.
// One launch serves up to three consecutive column segments of the partial rows, each with its own destination (e.g. the
// w2 | b1 | b2 gradients of project_bwd's 386-column rows).  Block = 32 columns x 32 row groups: thread (tx, ty) adds rows
// ty, ty + 32, .. with all its loads in flight (the first version had 8 row groups and ~37 dependent loads per thread:
// 14.5 us per launch, 16 launches per training step), the 32 group sums are then added in index order.
struct ReduceSeg {
  float* out[3];
  int n[3];
  int accumulate;   // 0: out = sum (no memset of the gradient needed), 1: out += sum (further batch chunks)
};
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const float* __restrict__ partial, int n_parts, int row_stride,
                                                               ReduceSeg seg) {
  __shared__ float red[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + tx;
  const int n_out = seg.n[0] + seg.n[1] + seg.n[2];
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (i < n_out) {
    int c = ty, u = 0;
    for (; c + 96 < n_parts; c += 128) {
#pragma unroll
      for (int k = 0; k < 4; ++k) s[k] += partial[static_cast<size_t>(c + 32 * k) * row_stride + i];
    }
    for (; c < n_parts; c += 32, ++u) s[u & 3] += partial[static_cast<size_t>(c) * row_stride + i];
  }
  red[ty][tx] = (s[0] + s[1]) + (s[2] + s[3]);
  __syncthreads();
  if (ty == 0 && i < n_out) {
    float t = red[0][tx];
#pragma unroll
    for (int r = 1; r < 32; ++r) t += red[r][tx];
    float* dst = i < seg.n[0] ? seg.out[0] + i
                 : (i < seg.n[0] + seg.n[1] ? seg.out[1] + (i - seg.n[0]) : seg.out[2] + (i - seg.n[0] - seg.n[1]));
    *dst = seg.accumulate ? *dst + t : t;
  }
}
cudaError_t launch_reduce_partials(const float* partial, int n_parts, int row_stride, float* out0, int n0, float* out1, int n1,
                                   float* out2, int n2, int accumulate, cudaStream_t stream) {
  const int n_out = n0 + n1 + n2;
  if (n_parts <= 0 || n_out <= 0) return cudaSuccess;
  ReduceSeg seg;
  seg.out[0] = out0; seg.out[1] = out1; seg.out[2] = out2;
  seg.n[0] = n0; seg.n[1] = n1; seg.n[2] = n2;
  seg.accumulate = accumulate;
  reduce_partials_kernel<<<(n_out + 31) / 32, 1024, 0, stream>>>(partial, n_parts, row_stride, seg);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- chan outer
// out[j][i] += sum_{b,pix} P[b][j][pix] * Q[b][i][pix];   rowsum[j] += sum_{b,pix} P[b][j][pix]
constexpr int kCoThreads = 256;

// 4 consecutive pixels of a staged row as fp32 (bf16 rows are widened by a shift)
template <typename T>
__device__ __forceinline__ float4 co_ld4(const unsigned char* row, int px);
template <>
__device__ __forceinline__ float4 co_ld4<float>(const unsigned char* row, int px) {
  return *reinterpret_cast<const float4*>(row + px * 4);
}
template <>
__device__ __forceinline__ float4 co_ld4<__nv_bfloat16>(const unsigned char* row, int px) {
  const uint2 v = *reinterpret_cast<const uint2*>(row + px * 2);
  return make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16),
                     __uint_as_float(v.y & 0xffff0000u));
}

// G[j][i] = sum_{b,pix} P[b][j][pix] Q[b][i][pix] and the row sums of P (the bias gradient): the 1x1-convolution weight
// gradients.  Round 1's version gave every thread a 2x2 (4x4) output tile: one 16-byte shared-memory read per 4 fma, so
// the kernel ran at the shared-memory rate, a quarter of the fma rate (68 / 98 us per launch at B = 64, 30 % of a
// training step).  Here a thread owns an 8 x 4 output tile (1.5 B of shared memory per fma) and the pixels of a chunk are
// split among NG thread groups whose partial tiles are added in a fixed order at the end; chunks arrive through a
// two-stage cp.async ring, so the loads of the next chunk overlap the arithmetic of the current one.
// Rows are assigned interleaved (j = a * NJ/8 + tj, i = c * NI/4 + ti) so that the rows a warp reads at the same time are
// consecutive and, with the 16-byte row skew, fall into different banks.
template <typename TP, typename TQ, int NJ, int NI>
struct CoCfg {
  static constexpr int TJ = 8, TI = 4;
  static constexpr int G = NJ * NI / (TJ * TI);          // threads per pixel group
  static constexpr int NG = kCoThreads / G;              // pixel groups
  static constexpr int PIX = (NJ >= 128) ? 64 : 128;     // pixels per chunk
  static constexpr int PXG = PIX / NG;                   // pixels per group and chunk
  static constexpr int NTI = NI / TI, NTJ = NJ / TJ;
  static constexpr int PITCH_P = PIX * static_cast<int>(sizeof(TP)) + 16, PITCH_Q = PIX * static_cast<int>(sizeof(TQ)) + 16;
  static constexpr int STAGE = NJ * PITCH_P + NI * PITCH_Q;
  static constexpr int OUT = NJ * NI + NJ;
  static constexpr size_t SMEM = (2 * STAGE > NG * OUT * 4) ? 2 * STAGE : NG * OUT * 4;
  static_assert(G * NG == kCoThreads && PXG % 4 == 0 && NJ % TJ == 0 && NI % TI == 0, "tile mismatch");
};

template <typename TP, typename TQ, int NJ, int NI>
__global__ void __launch_bounds__(kCoThreads)
    chan_outer_kernel(const TP* __restrict__ P, const TQ* __restrict__ Q, float* __restrict__ partial, int batch) {
  // partial[CTA][NJ*NI + NJ]: this CTA's share of G[j][i] and of the row sums sum_pix P[j][pix] (the bias gradient)
  using Cfg = CoCfg<TP, TQ, NJ, NI>;
  constexpr int TJ = Cfg::TJ, TI = Cfg::TI, PIX = Cfg::PIX;
  extern __shared__ __align__(16) unsigned char co_smem[];
  const int tid = threadIdx.x;
  const int grp = tid / Cfg::G, t = tid % Cfg::G;
  const int tj = t / Cfg::NTI, ti = t % Cfg::NTI;
  float acc[TJ][TI];
  float rs[TJ];
#pragma unroll
  for (int a = 0; a < TJ; ++a) {
    rs[a] = 0.f;
#pragma unroll
    for (int c = 0; c < TI; ++c) acc[a][c] = 0.f;
  }
  const int chunks = kHW / PIX;
  const int items = batch * chunks;
  auto stage_load = [&](int it, int st) {   // all threads: 16-byte cp.async pieces of the item's P and Q rows
    const int b = it / chunks, p0 = (it % chunks) * PIX;
    unsigned char* base = co_smem + st * Cfg::STAGE;
    constexpr int CP = PIX * static_cast<int>(sizeof(TP)) / 16, CQ = PIX * static_cast<int>(sizeof(TQ)) / 16;
    for (int e = tid; e < NJ * CP; e += kCoThreads) {
      const int j = e / CP, q = e % CP;
      const char* src = reinterpret_cast<const char*>(P + (static_cast<size_t>(b) * NJ + j) * kHW + p0) + q * 16;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(base + j * Cfg::PITCH_P + q * 16)), "l"(src) : "memory");
    }
    for (int e = tid; e < NI * CQ; e += kCoThreads) {
      const int i = e / CQ, q = e % CQ;
      const char* src = reinterpret_cast<const char*>(Q + (static_cast<size_t>(b) * NI + i) * kHW + p0) + q * 16;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(base + NJ * Cfg::PITCH_P + i * Cfg::PITCH_Q + q * 16)),
                   "l"(src) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  int n = 0;
  if (static_cast<int>(blockIdx.x) < items) stage_load(blockIdx.x, 0);
  for (int it = blockIdx.x; it < items; it += gridDim.x, ++n) {
    const int nxt = it + gridDim.x;
    if (nxt < items) {
      stage_load(nxt, (n + 1) & 1);   // the buffer was released by the barrier at the end of the previous iteration
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const unsigned char* ps = co_smem + (n & 1) * Cfg::STAGE;
    const unsigned char* qs = ps + NJ * Cfg::PITCH_P;
#pragma unroll 2
    for (int q = 0; q < Cfg::PXG / 4; ++q) {
      const int px = grp * Cfg::PXG + 4 * q;
      float4 pv[TJ], qv[TI];
#pragma unroll
      for (int a = 0; a < TJ; ++a) pv[a] = co_ld4<TP>(ps + (a * Cfg::NTJ + tj) * Cfg::PITCH_P, px);
#pragma unroll
      for (int c = 0; c < TI; ++c) qv[c] = co_ld4<TQ>(qs + (c * Cfg::NTI + ti) * Cfg::PITCH_Q, px);
#pragma unroll
      for (int a = 0; a < TJ; ++a) {
        if (ti == 0) rs[a] += (pv[a].x + pv[a].y) + (pv[a].z + pv[a].w);
#pragma unroll
        for (int c = 0; c < TI; ++c)
          acc[a][c] = fmaf(pv[a].x, qv[c].x, fmaf(pv[a].y, qv[c].y, fmaf(pv[a].z, qv[c].z, fmaf(pv[a].w, qv[c].w, acc[a][c]))));
      }
    }
    __syncthreads();   // everybody is done with this stage: the next iteration may refill it
  }
  // the NG pixel groups' tiles, added in group order (fixed summation tree)
  float* red = reinterpret_cast<float*>(co_smem);
#pragma unroll
  for (int a = 0; a < TJ; ++a) {
    const int j = a * Cfg::NTJ + tj;
#pragma unroll
    for (int c = 0; c < TI; ++c) red[grp * Cfg::OUT + j * NI + c * Cfg::NTI + ti] = acc[a][c];
    if (ti == 0) red[grp * Cfg::OUT + NJ * NI + j] = rs[a];
  }
  __syncthreads();
  float* prow = partial + static_cast<size_t>(blockIdx.x) * Cfg::OUT;
  for (int e = tid; e < Cfg::OUT; e += kCoThreads) {
    float v = red[e];
#pragma unroll
    for (int g = 1; g < Cfg::NG; ++g) v += red[g * Cfg::OUT + e];
    prow[e] = v;
  }
}

// returns the number of partial rows written (= grid size) through *n_parts
template <typename TP, typename TQ, int NJ, int NI>
cudaError_t launch_chan_outer(const void* P, const void* Q, float* partial, int* n_parts, int batch, cudaStream_t stream) {
  using Cfg = CoCfg<TP, TQ, NJ, NI>;
  auto kern = chan_outer_kernel<TP, TQ, NJ, NI>;
  constexpr size_t smem = Cfg::SMEM;
  static PerDeviceLaunch pd;
  cudaError_t e0 = per_device_setup(kern, smem, pd);
  if (e0 != cudaSuccess) return e0;
  const int items = batch * (kHW / Cfg::PIX);
  const int grid = items < 296 ? items : 296;   // 2 CTAs per SM; also the row count of the partial buffer
  kern<<<grid, kCoThreads, smem, stream>>>(static_cast<const TP*>(P), static_cast<const TQ*>(Q), partial, batch);
  *n_parts = grid;
  return cudaGetLastError();
}
template cudaError_t launch_chan_outer<float, float, 128, 32>(const void*, const void*, float*, int*, int, cudaStream_t);
template cudaError_t launch_chan_outer<float, __nv_bfloat16, 128, 32>(const void*, const void*, float*, int*, int, cudaStream_t);
template cudaError_t launch_chan_outer<float, float, 32, 32>(const void*, const void*, float*, int*, int, cudaStream_t);
template cudaError_t launch_chan_outer<float, __nv_bfloat16, 32, 32>(const void*, const void*, float*, int*, int, cudaStream_t);

// --------------------------------------------------------------------------------- spectral wgrad
// gWk[k][i][o] = sum_b conj(X[k][b][i]) * G[k][b][o];  one CTA per mode k, lane = o, warps split the batch.
constexpr int kSwWarps = 4;

__global__ void __launch_bounds__(kSwWarps * 32)
    spectral_wgrad_kernel(const float2* __restrict__ xm, const float2* __restrict__ gm, float2* __restrict__ gwk,
                          int batch) {
  __shared__ __align__(16) float2 xs[kSwWarps][kC];
  __shared__ __align__(16) float2 red[kSwWarps][kC][kC + 1];
  const int k = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2 acc_a[kC], acc_b[kC];  // a += xr*(gr,gi); b += xi*(gr,gi);  conj(x)*g = (a.x + b.y, a.y - b.x)
#pragma unroll
  for (int i = 0; i < kC; ++i) acc_a[i] = acc_b[i] = make_float2(0.f, 0.f);
  // the loads of the next three samples of this warp are in flight while the current one is multiplied (without the
  // prefetch every sample paid a full DRAM round trip: 44.7 us per launch at B = 256 for 38 MB)
  constexpr int kAhead = 3;
  float2 xq[kAhead], gq[kAhead];
#pragma unroll
  for (int u = 0; u < kAhead; ++u) {
    const int bu = warp + u * kSwWarps;
    if (bu < batch) {
      const size_t o = (static_cast<size_t>(k) * batch + bu) * kC + lane;
      xq[u] = __ldg(xm + o);
      gq[u] = __ldg(gm + o);
    }
  }
  for (int b = warp; b < batch; b += kSwWarps) {
    const int bn = b + kAhead * kSwWarps;
    float2 xn = make_float2(0.f, 0.f), gn = xn;
    if (bn < batch) {
      const size_t o = (static_cast<size_t>(k) * batch + bn) * kC + lane;
      xn = __ldg(xm + o);
      gn = __ldg(gm + o);
    }
    float2 xv, g;
    // rotating register queue with compile-time indices
    xv = xq[0]; g = gq[0];
#pragma unroll
    for (int u = 0; u < kAhead - 1; ++u) { xq[u] = xq[u + 1]; gq[u] = gq[u + 1]; }
    xq[kAhead - 1] = xn; gq[kAhead - 1] = gn;
    __syncwarp();
    xs[warp][lane] = xv;
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kC; i += 2) {
      const float4 v = *reinterpret_cast<const float4*>(&xs[warp][i]);
      acc_a[i] = ffma2(make_float2(v.x, v.x), g, acc_a[i]);
      acc_b[i] = ffma2(make_float2(v.y, v.y), g, acc_b[i]);
      acc_a[i + 1] = ffma2(make_float2(v.z, v.z), g, acc_a[i + 1]);
      acc_b[i + 1] = ffma2(make_float2(v.w, v.w), g, acc_b[i + 1]);
    }
  }
#pragma unroll
  for (int i = 0; i < kC; ++i) red[warp][i][lane] = make_float2(acc_a[i].x + acc_b[i].y, acc_a[i].y - acc_b[i].x);
  __syncthreads();
  for (int e = threadIdx.x; e < kC * kC; e += kSwWarps * 32) {
    const int i = e / kC, o = e % kC;
    float2 s = red[0][i][o];
#pragma unroll
    for (int w = 1; w < kSwWarps; ++w) {
      s.x += red[w][i][o].x;
      s.y += red[w][i][o].y;
    }
    gwk[static_cast<size_t>(k) * kC * kC + e] = s;
  }
}

cudaError_t launch_spectral_wgrad(const void* xm, const void* gm, void* gwk, int batch, cudaStream_t stream) {
  spectral_wgrad_kernel<<<kModes, kSwWarps * 32, 0, stream>>>(static_cast<const float2*>(xm), static_cast<const float2*>(gm),
                                                             static_cast<float2*>(gwk), batch);
  return cudaGetLastError();
}

// --------------------------------------------------------------------------------------- lift bwd
// g_w[c][q] (q<5: u,v,mask,x,y; q>=5: case params), g_b[c] from d a0.  One CTA per (channel c, sample
// slice); per-sample plane sums T[b][c] carry the bias and case-parameter columns.
constexpr int kLbThreads = 256;

__global__ void __launch_bounds__(kLbThreads)
    lift_bwd_kernel(const float* __restrict__ da0,     // [B][32][4096]
                    const float* __restrict__ inputs,  // [B][2][4096]
                    const float* __restrict__ mask,    // [B][4096]
                    const float* __restrict__ params,  // [B][p]
                    const float* __restrict__ gx, const float* __restrict__ gy, float* __restrict__ partial,
                    int batch, int p) {   // partial[blockIdx.y][c][nin + 1]: weight row of channel c, then its bias
  // Every thread accumulates its share of all six sums over ALL its samples (the case-parameter columns are linear in the
  // per-sample plane sum, so its per-thread part is weighted by params[b][q] on the fly); one block reduction at the end.
  // (Round 1 reduced over the block after every sample: two barriers per 16 KB plane, 80 us at B = 256 for 134 MB.)
  __shared__ float red[kLbThreads / 32][6 + kMaxCaseParams];
  const int c = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nin = 5 + p;
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float gp_acc[kMaxCaseParams];
#pragma unroll
  for (int q = 0; q < kMaxCaseParams; ++q) gp_acc[q] = 0.f;
  for (int b = blockIdx.y; b < batch; b += gridDim.y) {
    const float* d = da0 + (static_cast<size_t>(b) * kC + c) * kHW;
    float dplane = 0.f;   // this thread's share of the plane sum of sample b
#pragma unroll 4
    for (int px = tid * 4; px < kHW; px += kLbThreads * 4) {
      const float4 dv = *reinterpret_cast<const float4*>(d + px);
      const float4 u = *reinterpret_cast<const float4*>(inputs + (static_cast<size_t>(b) * 2 + 0) * kHW + px);
      const float4 v = *reinterpret_cast<const float4*>(inputs + (static_cast<size_t>(b) * 2 + 1) * kHW + px);
      const float4 m = *reinterpret_cast<const float4*>(mask + static_cast<size_t>(b) * kHW + px);
      const float4 yw = *reinterpret_cast<const float4*>(gy + (px & 63));
      const float xh = gx[px >> 6];
      const float dsum = (dv.x + dv.y) + (dv.z + dv.w);
      s[0] += dv.x * u.x + dv.y * u.y + dv.z * u.z + dv.w * u.w;
      s[1] += dv.x * v.x + dv.y * v.y + dv.z * v.z + dv.w * v.w;
      s[2] += dv.x * m.x + dv.y * m.y + dv.z * m.z + dv.w * m.w;
      s[3] += dsum * xh;
      s[4] += dv.x * yw.x + dv.y * yw.y + dv.z * yw.z + dv.w * yw.w;
      dplane += dsum;
    }
    s[5] += dplane;
#pragma unroll
    for (int q = 0; q < kMaxCaseParams; ++q)
      if (q < p) gp_acc[q] = fmaf(dplane, params[b * p + q], gp_acc[q]);
  }
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    const float r = warp_sum(s[q]);
    if (lane == 0) red[warp][q] = r;
  }
#pragma unroll
  for (int q = 0; q < kMaxCaseParams; ++q) {
    const float r = warp_sum(gp_acc[q]);
    if (lane == 0) red[warp][6 + q] = r;
  }
  __syncthreads();
  if (tid < 6 + kMaxCaseParams) {
    float t = 0.f;
    for (int w = 0; w < kLbThreads / 32; ++w) t += red[w][tid];   // warp order: fixed
    float* prow = partial + (static_cast<size_t>(blockIdx.y) * kC + c) * (nin + 1);
    if (tid < 5) prow[tid] = t;
    else if (tid == 5) prow[nin] = t;
    else if (tid - 6 < p) prow[5 + tid - 6] = t;
  }
}

// g_w[c][q] = sum_y partial[y][c][q], g_b[c] = sum_y partial[y][c][nin]   (fixed order); kAccum: += instead of =
template <bool kAccum>
__global__ void lift_bwd_reduce_kernel(const float* __restrict__ partial, int n_parts, int nin, float* __restrict__ g_w,
                                       float* __restrict__ g_b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kC * (nin + 1)) return;
  const int c = i / (nin + 1), q = i % (nin + 1);
  float s = 0.f;
  for (int y = 0; y < n_parts; ++y) s += partial[(static_cast<size_t>(y) * kC + c) * (nin + 1) + q];
  float* dst = q < nin ? g_w + c * nin + q : g_b + c;
  if constexpr (kAccum) *dst += s;   // a later step of the rollout backward's sweep
  else *dst = s;                     // the only contribution: no memset of the gradient needed
}

cudaError_t launch_lift_bwd(const float* da0, const float* inputs, const float* mask, const float* params,
                            const float* gx, const float* gy, float* g_w, float* g_b, float* partial, int batch, int p,
                            int accumulate, cudaStream_t stream) {
  if (p < 0 || p > kMaxCaseParams) return cudaErrorInvalidValue;
  dim3 grid(kC, batch < 16 ? batch : 16);
  lift_bwd_kernel<<<grid, kLbThreads, 0, stream>>>(da0, inputs, mask, params, gx, gy, partial, batch, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int n = kC * (5 + p + 1);
  auto reduce = accumulate ? lift_bwd_reduce_kernel<true> : lift_bwd_reduce_kernel<false>;
  reduce<<<(n + 127) / 128, 128, 0, stream>>>(partial, static_cast<int>(grid.y), 5 + p, g_w, g_b);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------- lift bwd (data)
// The data adjoint of the lift (gradients w.r.t. the input frame and the case parameters):
//   d_inputs[b][c][pix] = sum_o fc0_w[o][c] d_a0[b][o][pix]                  c = 0 (u), 1 (v)
//   d_params[b][j]      = sum_o fc0_w[o][5 + j] sum_pix d_a0[b][o][pix]
// One CTA owns one sample, so the plane sums are block reductions in a fixed order (warp butterflies, then warps in
// index order): no atomics, bit-reproducible.  Thread = kLdVec groups of 4 consecutive pixels, 16-byte loads and stores;
// the case-parameter weights are applied to each thread's per-channel pixel sum on the fly, so only p values per thread
// are reduced at the end.  One pass over d_a0 (float32 in both storage modes, 134 MB at B = 256).
// kHandOff (the rollout backward's sweep): d_inputs = (sum_o fc0_w[o][c] d_a0) + add, where `add` (or null) is the
// upstream gradient of the previous step's prediction, so d_inputs becomes that step's whole upstream gradient in this
// one pass; d_params += instead of = (the case parameters feed every step).  `gate` (or null; kHandOff only, teacher
// forcing): where gate[b] != 0 the previous prediction was not fed to this step, so d_inputs = add, a copy bit for bit
// (nothing of d_a0, a NaN included, reaches it); d_params still takes the step's share.
constexpr int kLdThreads = 512;
constexpr int kLdVec = kHW / (4 * kLdThreads);   // float4 groups per thread and channel

template <bool kHandOff>
__global__ void __launch_bounds__(kLdThreads)
    lift_bwd_data_kernel(const float* __restrict__ da0,     // [B][32][4096]
                         const float* __restrict__ fc0_w,   // [32][5+p]
                         float* __restrict__ d_inputs,      // [B][2][4096] or null
                         float* __restrict__ d_params,      // [B][p] or null
                         const float* __restrict__ add,     // [B][2][4096] or null (kHandOff only)
                         const unsigned char* __restrict__ gate,   // [B] or null (kHandOff only)
                         int p) {
  __shared__ float wu[kC], wv[kC];
  __shared__ __align__(16) float wp[kC][kMaxCaseParams];   // columns 5..5+p, zero-padded to 16
  __shared__ float red[kLdThreads / 32][kMaxCaseParams];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x;
  const int nin = 5 + p;
  if (tid < kC) {
    wu[tid] = fc0_w[tid * nin];
    wv[tid] = fc0_w[tid * nin + 1];
  }
  for (int e = tid; e < kC * kMaxCaseParams; e += kLdThreads) {
    const int o = e / kMaxCaseParams, j = e % kMaxCaseParams;
    wp[o][j] = j < p ? fc0_w[o * nin + 5 + j] : 0.f;
  }
  __syncthreads();

  const float4* d = reinterpret_cast<const float4*>(da0 + static_cast<size_t>(b) * kC * kHW);
  const bool want_p = d_params != nullptr;
  float4 du[kLdVec], dv[kLdVec];
  float cp[kMaxCaseParams];
#pragma unroll
  for (int k = 0; k < kLdVec; ++k) du[k] = dv[k] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int j = 0; j < kMaxCaseParams; ++j) cp[j] = 0.f;
#pragma unroll 4
  for (int o = 0; o < kC; ++o) {
    const float a = wu[o], c = wv[o];
    float s = 0.f;   // this thread's share of the plane sum of channel o
#pragma unroll
    for (int k = 0; k < kLdVec; ++k) {
      const float4 x = __ldcs(d + o * (kHW / 4) + k * kLdThreads + tid);   // last use of d_a0: stream through L2
      du[k].x = fmaf(a, x.x, du[k].x); du[k].y = fmaf(a, x.y, du[k].y);
      du[k].z = fmaf(a, x.z, du[k].z); du[k].w = fmaf(a, x.w, du[k].w);
      dv[k].x = fmaf(c, x.x, dv[k].x); dv[k].y = fmaf(c, x.y, dv[k].y);
      dv[k].z = fmaf(c, x.z, dv[k].z); dv[k].w = fmaf(c, x.w, dv[k].w);
      s += (x.x + x.y) + (x.z + x.w);
    }
    if (want_p) {
      const float4* wrow = reinterpret_cast<const float4*>(&wp[o][0]);
#pragma unroll
      for (int q = 0; q < kMaxCaseParams / 4; ++q) {
        const float4 t = wrow[q];
        cp[4 * q] = fmaf(t.x, s, cp[4 * q]);
        cp[4 * q + 1] = fmaf(t.y, s, cp[4 * q + 1]);
        cp[4 * q + 2] = fmaf(t.z, s, cp[4 * q + 2]);
        cp[4 * q + 3] = fmaf(t.w, s, cp[4 * q + 3]);
      }
    }
  }
  if (d_inputs != nullptr) {
    float4* u_out = reinterpret_cast<float4*>(d_inputs + static_cast<size_t>(b) * 2 * kHW);
    float4* v_out = u_out + kHW / 4;
    if constexpr (kHandOff) {
      if (add != nullptr) {
        const float4* u_add = reinterpret_cast<const float4*>(add + static_cast<size_t>(b) * 2 * kHW);
        const float4* v_add = u_add + kHW / 4;
        if (gate != nullptr && gate[b] != 0) {   // a forced sample: the carry is add alone
#pragma unroll
          for (int k = 0; k < kLdVec; ++k) {
            du[k] = __ldcs(u_add + k * kLdThreads + tid);
            dv[k] = __ldcs(v_add + k * kLdThreads + tid);
          }
        } else {
#pragma unroll
          for (int k = 0; k < kLdVec; ++k) {
            const float4 a = __ldcs(u_add + k * kLdThreads + tid), c = __ldcs(v_add + k * kLdThreads + tid);
            du[k].x += a.x; du[k].y += a.y; du[k].z += a.z; du[k].w += a.w;
            dv[k].x += c.x; dv[k].y += c.y; dv[k].z += c.z; dv[k].w += c.w;
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kLdVec; ++k) {
      u_out[k * kLdThreads + tid] = du[k];
      v_out[k * kLdThreads + tid] = dv[k];
    }
  }
  if (want_p) {
#pragma unroll
    for (int j = 0; j < kMaxCaseParams; ++j) {
      if (j < p) {
        const float r = warp_sum(cp[j]);
        if (lane == 0) red[warp][j] = r;
      }
    }
    __syncthreads();
    if (tid < p) {
      float t = 0.f;
      for (int w = 0; w < kLdThreads / 32; ++w) t += red[w][tid];   // warp order: fixed
      if constexpr (kHandOff) d_params[static_cast<size_t>(b) * p + tid] += t;
      else d_params[static_cast<size_t>(b) * p + tid] = t;
    }
  }
}

// hand_off = 0: the single-step data adjoint (d_inputs, d_params written; `add` and `gate` must be null).  hand_off = 1:
// the rollout sweep's mode described above the kernel.
cudaError_t launch_lift_bwd_data(const float* da0, const float* fc0_w, float* d_inputs, float* d_params, const float* add,
                                 int hand_off, int batch, int p, cudaStream_t stream, const unsigned char* gate) {
  if (p < 0 || p > kMaxCaseParams) return cudaErrorInvalidValue;
  if (p == 0) d_params = nullptr;
  if (d_inputs == nullptr && d_params == nullptr) return cudaSuccess;
  if (hand_off)
    lift_bwd_data_kernel<true><<<batch, kLdThreads, 0, stream>>>(da0, fc0_w, d_inputs, d_params, add, gate, p);
  else
    lift_bwd_data_kernel<false><<<batch, kLdThreads, 0, stream>>>(da0, fc0_w, d_inputs, d_params, nullptr, nullptr, p);
  return cudaGetLastError();
}

}  // namespace fno
