// SURVEY.md 8f.1 -- rollout evaluation metrics on the device.
// The reference computes, per rollout step and per case, mse / nmse / mae of the masked u channel with three
// .item() host syncs each (src/test_multistep.py:73-83, 153-177).  Here one launch reduces every (step, case) plane
// to the three sums the metrics are made of; a single D2H of steps*B*3 floats replaces 3*steps*B synchronisations.
#include "fno_common.cuh"

namespace fno {

constexpr int kMtThreads = 256;

// The per-plane reduction of every rollout-metrics kernel (multistep_metrics_kernel, grid_multistep_metrics_kernel,
// window_metrics_kernel), one function so that their sums agree bit for bit on the same pixels.  A plane is n_items
// items of kVec consecutive pixels; thread t takes items t, t + 256, ..., and `load(i, pp, ll)` gives item i's masked
// predictions and labels.  Per pixel, in order: d = pp - ll, se = fmaf(d, d, se), sl = fmaf(ll, ll, sl), sa += |d|;
// then the xor shuffle tree and the eight warps added in a fixed order (no atomics: a repeated launch is bit-identical).
// out[plane][0..2] = (sum d^2, sum ll^2, sum |d|).
template <int kVec, typename Load>
__device__ __forceinline__ void reduce_plane_sums(int n_items, Load load, float* __restrict__ out, size_t plane) {
  __shared__ float red[kMtThreads / 32][3];
  float se = 0.f, sl = 0.f, sa = 0.f;
  for (int i = threadIdx.x; i < n_items; i += kMtThreads) {
    float pp[kVec], ll[kVec];
    load(i, pp, ll);
#pragma unroll
    for (int c = 0; c < kVec; ++c) {
      const float d = pp[c] - ll[c];
      se = fmaf(d, d, se);
      sl = fmaf(ll[c], ll[c], sl);
      sa += fabsf(d);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sl += __shfl_xor_sync(0xffffffffu, sl, o);
    sa += __shfl_xor_sync(0xffffffffu, sa, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    red[warp][0] = se;
    red[warp][1] = sl;
    red[warp][2] = sa;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kMtThreads / 32; ++w) t += red[w][threadIdx.x];  // fixed order: deterministic
    out[plane * 3 + threadIdx.x] = t;
  }
}

// preds_seq [S][B][2][64][64] (channel 0 = u), label_u [S][B][64][64], mask [S][B][64][64]
// out [S][B][3] = (sum (p-l)^2, sum l^2, sum |p-l|) over the 4096 pixels, with p, l multiplied by the mask
__global__ void __launch_bounds__(kMtThreads)
    multistep_metrics_kernel(const float* __restrict__ preds_seq, const float* __restrict__ label_u,
                             const float* __restrict__ mask, float* __restrict__ out, int batch) {
  const int b = blockIdx.x, s = blockIdx.y;
  const size_t plane = static_cast<size_t>(s) * batch + b;
  const float4* p = reinterpret_cast<const float4*>(preds_seq + plane * 2 * kHW);
  const float4* l = reinterpret_cast<const float4*>(label_u + plane * kHW);
  const float4* m = reinterpret_cast<const float4*>(mask + plane * kHW);
  reduce_plane_sums<4>(kHW / 4, [&](int i, float (&pp)[4], float (&ll)[4]) {
    const float4 pv = __ldg(p + i), lv = __ldg(l + i), mv = __ldg(m + i);
    pp[0] = pv.x * mv.x, pp[1] = pv.y * mv.y, pp[2] = pv.z * mv.z, pp[3] = pv.w * mv.w;
    ll[0] = lv.x * mv.x, ll[1] = lv.y * mv.y, ll[2] = lv.z * mv.z, ll[3] = lv.w * mv.w;
  }, out, plane);
}

cudaError_t launch_multistep_metrics(const float* preds_seq, const float* label_u, const float* mask, float* out,
                                     int steps, int batch, cudaStream_t stream) {
  dim3 grid(batch, steps);
  multistep_metrics_kernel<<<grid, kMtThreads, 0, stream>>>(preds_seq, label_u, mask, out, batch);
  return cudaGetLastError();
}

}  // namespace fno

// ------------------------------------------------------------------------------------------------
// SURVEY.md 8f.2 -- device-resident input pipeline.  The reference keeps every (input, label) frame pair of the
// training set in host tensors (src/dataset/cavity.py:326-331), and per batch runs DataLoader indexing, torch.stack,
// three channel slices, a Python loop over the case-parameter dicts and four .cuda() copies
// (collate_fn, src/train_auto.py:33-58).  With the frames resident in HBM one launch gathers a batch:
//   inputs[b] = frames_in[idx[b]][0:2], mask[b] = frames_in[idx[b]][2], label[b] = frames_out[idx[b]][0:2],
//   case_params[b] = case_table[case_ids[idx[b]]]
// ------------------------------------------------------------------------------------------------
namespace fno {

template <typename TFrame>
__device__ __forceinline__ float4 gather_ld4(const TFrame* p);
template <>
__device__ __forceinline__ float4 gather_ld4<float>(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
template <>
__device__ __forceinline__ float4 gather_ld4<__nv_bfloat16>(const __nv_bfloat16* p) {
  const uint2 raw = __ldg(reinterpret_cast<const uint2*>(p));
  const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&raw.x), hi = *reinterpret_cast<const __nv_bfloat162*>(&raw.y);
  const float2 a = __bfloat1622float2(lo), b = __bfloat1622float2(hi);
  return make_float4(a.x, a.y, b.x, b.y);
}

constexpr int kGbThreads = 256;

// grid (5 planes, n_idx): plane 0,1 -> inputs u,v; 2 -> mask; 3,4 -> label u,v
template <typename TFrame>
__global__ void __launch_bounds__(kGbThreads)
    gather_batch_kernel(const TFrame* __restrict__ frames_in, const TFrame* __restrict__ frames_out,
                        const float* __restrict__ case_table, const int* __restrict__ case_ids,
                        const long long* __restrict__ idx, int n_case_params, float* __restrict__ inputs,
                        float* __restrict__ label, float* __restrict__ mask, float* __restrict__ case_params) {
  const int plane = blockIdx.x, b = blockIdx.y;
  const long long i = idx[b];
  const TFrame* src = (plane < 3 ? frames_in : frames_out) + (static_cast<size_t>(i) * 3 + (plane < 3 ? plane : plane - 3)) * kHW;
  float* dst = plane < 2   ? inputs + (static_cast<size_t>(b) * 2 + plane) * kHW
               : plane == 2 ? mask + static_cast<size_t>(b) * kHW
                            : label + (static_cast<size_t>(b) * 2 + (plane - 3)) * kHW;
  for (int e = threadIdx.x * 4; e < kHW; e += kGbThreads * 4)
    *reinterpret_cast<float4*>(dst + e) = gather_ld4<TFrame>(src + e);
  if (plane == 0 && threadIdx.x < n_case_params)
    case_params[static_cast<size_t>(b) * n_case_params + threadIdx.x] =
        __ldg(case_table + static_cast<size_t>(case_ids[i]) * n_case_params + threadIdx.x);
}

cudaError_t launch_gather_batch(const void* frames_in, const void* frames_out, const float* case_table, const int* case_ids,
                                const long long* idx, int n_idx, int n_case_params, int frame_bf16, float* inputs,
                                float* label, float* mask, float* case_params, cudaStream_t stream) {
  dim3 grid(5, n_idx);
  if (frame_bf16)
    gather_batch_kernel<__nv_bfloat16><<<grid, kGbThreads, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(frames_in), static_cast<const __nv_bfloat16*>(frames_out), case_table, case_ids, idx,
        n_case_params, inputs, label, mask, case_params);
  else
    gather_batch_kernel<float><<<grid, kGbThreads, 0, stream>>>(static_cast<const float*>(frames_in),
                                                                static_cast<const float*>(frames_out), case_table, case_ids,
                                                                idx, n_case_params, inputs, label, mask, case_params);
  return cudaGetLastError();
}

}  // namespace fno

// ------------------------------------------------------------------------------------------------
// Grid-generic versions of the two kernels above, for any H x W the grid path runs (24..128 each; the tube and dam
// problems' 66x65).  A plane of H*W floats (or bf16) need not start on more than an element boundary -- a 66x65 fp32
// plane is 17,160 B, so every odd plane of label_u / mask is only 8-byte aligned, and at odd H*W (25x127) only 4-byte
// aligned -- so both kernels use scalar loads and stores.  They move a few MB per call; the loads are not the limit.
// ------------------------------------------------------------------------------------------------
namespace fno {

// Same layouts and sums as multistep_metrics_kernel with hw = H*W in place of 4096, one pixel per item.  grid (B, S): one
// CTA per (step, case) plane.
__global__ void __launch_bounds__(kMtThreads)
    grid_multistep_metrics_kernel(const float* __restrict__ preds_seq, const float* __restrict__ label_u,
                                  const float* __restrict__ mask, float* __restrict__ out, int batch, int hw) {
  const int b = blockIdx.x, s = blockIdx.y;
  const size_t plane = static_cast<size_t>(s) * batch + b;
  const float* p = preds_seq + plane * 2 * hw;   // channel 0 = u
  const float* l = label_u + plane * hw;
  const float* m = mask + plane * hw;
  reduce_plane_sums<1>(hw, [&](int i, float (&pp)[1], float (&ll)[1]) {
    const float mv = __ldg(m + i);
    pp[0] = __ldg(p + i) * mv, ll[0] = __ldg(l + i) * mv;
  }, out, plane);
}

cudaError_t launch_grid_multistep_metrics(const float* preds_seq, const float* label_u, const float* mask, float* out,
                                          int steps, int batch, int h, int w, cudaStream_t stream) {
  dim3 grid(batch, steps);
  grid_multistep_metrics_kernel<<<grid, kMtThreads, 0, stream>>>(preds_seq, label_u, mask, out, batch, h * w);
  return cudaGetLastError();
}

// Single-step evaluation (reference src/train_auto.py:61-148, `evaluate`): per sample b of a (B, 2, H, W) batch
//   out[b][0..2] = sum (p - l*m)^2, sum |p - l*m|, sum (l*m)^2        both channels, p = preds as the model returns them
//                                                                      (already masked), m broadcast over the channels
//   out[b][3..5] = sum (x_u - l_u)^2, sum |x_u - l_u|, sum l_u^2       channel 0 of inputs / label, no mask
// i.e. the terms of the model's loss on (preds, label * mask) and of the input loss on (inputs[:, :1], label[:, :1]).
// grid (B): one CTA per sample, scalar loads (caller tensors, planes only 4-byte aligned at odd H*W), each thread's
// pixels, the shuffle tree and the warp order fixed: a repeated launch is bit-identical (no atomics).
constexpr int kEvThreads = 256;

__global__ void __launch_bounds__(kEvThreads)
    eval_sums_kernel(const float* __restrict__ preds, const float* __restrict__ label, const float* __restrict__ mask,
                     const float* __restrict__ inputs, float* __restrict__ out, int hw) {
  __shared__ float red[kEvThreads / 32][6];
  const size_t b = blockIdx.x;
  const float* p = preds + b * 2 * hw;
  const float* l = label + b * 2 * hw;
  const float* x = inputs + b * 2 * hw;   // channel 0 = u
  const float* m = mask + b * hw;
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = threadIdx.x; i < hw; i += kEvThreads) {
    const float mv = __ldg(m + i);
    const float p0 = __ldg(p + i), p1 = __ldg(p + hw + i);
    const float l0 = __ldg(l + i), l1 = __ldg(l + hw + i);
    const float x0 = __ldg(x + i);
    const float lm0 = l0 * mv, lm1 = l1 * mv;
    const float d0 = p0 - lm0, d1 = p1 - lm1, du = x0 - l0;
    s[0] = fmaf(d1, d1, fmaf(d0, d0, s[0]));
    s[1] += fabsf(d0) + fabsf(d1);
    s[2] = fmaf(lm1, lm1, fmaf(lm0, lm0, s[2]));
    s[3] = fmaf(du, du, s[3]);
    s[4] += fabsf(du);
    s[5] = fmaf(l0, l0, s[5]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < 6; ++k) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < 6; ++k) red[warp][k] = s[k];
  __syncthreads();
  if (threadIdx.x < 6) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kEvThreads / 32; ++w) t += red[w][threadIdx.x];  // fixed order: deterministic
    out[b * 6 + threadIdx.x] = t;
  }
}

cudaError_t launch_eval_sums(const float* preds, const float* label, const float* mask, const float* inputs, float* out,
                             int batch, int h, int w, cudaStream_t stream) {
  eval_sums_kernel<<<batch, kEvThreads, 0, stream>>>(preds, label, mask, inputs, out, h * w);
  return cudaGetLastError();
}

__device__ __forceinline__ float frame_ld(const float* p) { return __ldg(p); }
__device__ __forceinline__ float frame_ld(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }

// Same job as gather_batch_kernel at hw = H*W.  grid (n_idx, 5 planes): plane 0,1 -> inputs u,v; 2 -> mask;
// 3,4 -> label u,v.  The batch index is on x so that n_idx is not held to gridDim.y's 65,535.
template <typename TFrame>
__global__ void __launch_bounds__(kGbThreads)
    grid_gather_batch_kernel(const TFrame* __restrict__ frames_in, const TFrame* __restrict__ frames_out,
                             const float* __restrict__ case_table, const int* __restrict__ case_ids,
                             const long long* __restrict__ idx, int n_case_params, int hw, float* __restrict__ inputs,
                             float* __restrict__ label, float* __restrict__ mask, float* __restrict__ case_params) {
  const int b = blockIdx.x, plane = blockIdx.y;
  const long long i = idx[b];
  const TFrame* src = (plane < 3 ? frames_in : frames_out) + (static_cast<size_t>(i) * 3 + (plane < 3 ? plane : plane - 3)) * hw;
  float* dst = plane < 2   ? inputs + (static_cast<size_t>(b) * 2 + plane) * hw
               : plane == 2 ? mask + static_cast<size_t>(b) * hw
                            : label + (static_cast<size_t>(b) * 2 + (plane - 3)) * hw;
  for (int e = threadIdx.x; e < hw; e += kGbThreads) dst[e] = frame_ld(src + e);
  if (plane == 0 && threadIdx.x < n_case_params)
    case_params[static_cast<size_t>(b) * n_case_params + threadIdx.x] =
        __ldg(case_table + static_cast<size_t>(case_ids[i]) * n_case_params + threadIdx.x);
}

cudaError_t launch_grid_gather_batch(const void* frames_in, const void* frames_out, const float* case_table,
                                     const int* case_ids, const long long* idx, int n_idx, int n_case_params,
                                     int frame_bf16, float* inputs, float* label, float* mask, float* case_params, int h,
                                     int w, cudaStream_t stream) {
  dim3 grid(n_idx, 5);
  if (frame_bf16)
    grid_gather_batch_kernel<__nv_bfloat16><<<grid, kGbThreads, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(frames_in), static_cast<const __nv_bfloat16*>(frames_out), case_table, case_ids,
        idx, n_case_params, h * w, inputs, label, mask, case_params);
  else
    grid_gather_batch_kernel<float><<<grid, kGbThreads, 0, stream>>>(
        static_cast<const float*>(frames_in), static_cast<const float*>(frames_out), case_table, case_ids, idx,
        n_case_params, h * w, inputs, label, mask, case_params);
  return cudaGetLastError();
}

}  // namespace fno

// ------------------------------------------------------------------------------------------------
// Window gather for training through K-step rollouts (cfdbench_b200.train_auto with rollout_steps = K).  A dataset holds
// a case's samples contiguously with inputs = frames[:-s], labels = frames[s:] (s = time_step_size), so the k-th target of
// the window that starts at sample j is labels[j + k s].  One launch gathers the start samples as the gathers above do and
// the K masked targets of each window:
//   inputs, label, mask, case_params as gather_batch_kernel / grid_gather_batch_kernel for the same idx (label is skipped
//   when null), labels_seq[k][b][c] = frames_out[idx[b] + k s][c] * frames_in[idx[b]][2]   (c = u, v; one fp32 multiply,
//   so it equals label * mask bit for bit).
// A window that runs past n_frames is not read and none of its sample's outputs are written, the guard style of the
// step-cursor kernels.  grid (n_idx, 5 + 2 steps): plane 0,1 -> inputs; 2 -> mask; 3,4 -> label; 5 + 2k + c -> labels_seq.
// kVec: 64x64 frames, 16-byte accesses as gather_batch_kernel; otherwise scalar accesses (see the grid section's header).
// ------------------------------------------------------------------------------------------------
namespace fno {

template <typename TFrame, bool kVec>
__global__ void __launch_bounds__(kGbThreads)
    gather_window_kernel(const TFrame* __restrict__ frames_in, const TFrame* __restrict__ frames_out,
                         const float* __restrict__ case_table, const int* __restrict__ case_ids,
                         const long long* __restrict__ idx, int n_idx, int n_case_params, int hw, int steps,
                         int time_step_size, long long n_frames, float* __restrict__ inputs, float* __restrict__ label,
                         float* __restrict__ mask, float* __restrict__ case_params, float* __restrict__ labels_seq) {
  const int b = blockIdx.x, plane = blockIdx.y;
  const long long i = idx[b];
  if (i < 0 || i + static_cast<long long>(steps - 1) * time_step_size >= n_frames) return;
  const TFrame* src;
  const TFrame* msk = nullptr;
  float* dst;
  if (plane < 3) {
    src = frames_in + (static_cast<size_t>(i) * 3 + plane) * hw;
    dst = plane < 2 ? inputs + (static_cast<size_t>(b) * 2 + plane) * hw : mask + static_cast<size_t>(b) * hw;
  } else if (plane < 5) {
    if (label == nullptr) return;
    src = frames_out + (static_cast<size_t>(i) * 3 + (plane - 3)) * hw;
    dst = label + (static_cast<size_t>(b) * 2 + (plane - 3)) * hw;
  } else {
    const int k = (plane - 5) >> 1, c = (plane - 5) & 1;
    src = frames_out + ((static_cast<size_t>(i) + static_cast<size_t>(k) * time_step_size) * 3 + c) * hw;
    msk = frames_in + (static_cast<size_t>(i) * 3 + 2) * hw;
    dst = labels_seq + ((static_cast<size_t>(k) * n_idx + b) * 2 + c) * hw;
  }
  if constexpr (kVec) {
    for (int e = threadIdx.x * 4; e < kHW; e += kGbThreads * 4) {
      float4 v = gather_ld4<TFrame>(src + e);
      if (msk) {
        const float4 m = gather_ld4<TFrame>(msk + e);
        v.x *= m.x;
        v.y *= m.y;
        v.z *= m.z;
        v.w *= m.w;
      }
      *reinterpret_cast<float4*>(dst + e) = v;
    }
  } else {
    for (int e = threadIdx.x; e < hw; e += kGbThreads) dst[e] = msk ? frame_ld(src + e) * frame_ld(msk + e) : frame_ld(src + e);
  }
  if (plane == 0 && threadIdx.x < n_case_params)
    case_params[static_cast<size_t>(b) * n_case_params + threadIdx.x] =
        __ldg(case_table + static_cast<size_t>(case_ids[i]) * n_case_params + threadIdx.x);
}

template <bool kVec>
static cudaError_t launch_gather_window_impl(const void* frames_in, const void* frames_out, const float* case_table,
                                             const int* case_ids, const long long* idx, int n_idx, int n_case_params,
                                             int frame_bf16, float* inputs, float* label, float* mask, float* case_params,
                                             int steps, int time_step_size, long long n_frames, float* labels_seq, int hw,
                                             cudaStream_t stream) {
  dim3 grid(n_idx, 5 + 2 * steps);
  if (frame_bf16)
    gather_window_kernel<__nv_bfloat16, kVec><<<grid, kGbThreads, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(frames_in), static_cast<const __nv_bfloat16*>(frames_out), case_table, case_ids,
        idx, n_idx, n_case_params, hw, steps, time_step_size, n_frames, inputs, label, mask, case_params, labels_seq);
  else
    gather_window_kernel<float, kVec><<<grid, kGbThreads, 0, stream>>>(
        static_cast<const float*>(frames_in), static_cast<const float*>(frames_out), case_table, case_ids, idx, n_idx,
        n_case_params, hw, steps, time_step_size, n_frames, inputs, label, mask, case_params, labels_seq);
  return cudaGetLastError();
}

cudaError_t launch_gather_window(const void* frames_in, const void* frames_out, const float* case_table, const int* case_ids,
                                 const long long* idx, int n_idx, int n_case_params, int frame_bf16, float* inputs,
                                 float* label, float* mask, float* case_params, int steps, int time_step_size,
                                 long long n_frames, float* labels_seq, cudaStream_t stream) {
  return launch_gather_window_impl<true>(frames_in, frames_out, case_table, case_ids, idx, n_idx, n_case_params, frame_bf16,
                                         inputs, label, mask, case_params, steps, time_step_size, n_frames, labels_seq, kHW,
                                         stream);
}
cudaError_t launch_grid_gather_window(const void* frames_in, const void* frames_out, const float* case_table,
                                      const int* case_ids, const long long* idx, int n_idx, int n_case_params,
                                      int frame_bf16, float* inputs, float* label, float* mask, float* case_params,
                                      int steps, int time_step_size, long long n_frames, float* labels_seq, int h, int w,
                                      cudaStream_t stream) {
  return launch_gather_window_impl<false>(frames_in, frames_out, case_table, case_ids, idx, n_idx, n_case_params,
                                          frame_bf16, inputs, label, mask, case_params, steps, time_step_size, n_frames,
                                          labels_seq, h * w, stream);
}

}  // namespace fno

// ------------------------------------------------------------------------------------------------
// Rollout metrics of the windows of a device-resident split (cfdbench_b200.evaluate_rollout_auto).  Step k (0-based) of
// the window that starts at sample j = starts[b] is compared with the true frame k steps on, frames_out[j + k s]
// (s = time_step_size), u channel only, both sides multiplied by the start sample's mask frames_in[j][2] -- the mask the
// inference rollout applies to its predictions:
//   out[k][b][0..2] = (sum (p-l)^2, sum l^2, sum |p-l|),  p = preds_seq[k][b][0] * m,  l = frames_out[j + k s][0] * m.
// The sums are reduce_plane_sums', so they equal fno_[grid_]multistep_metrics' on the gathered (label_u, mask) bit for
// bit, without the (S, B, H, W) label and mask sequences: only the u plane of each target and the start mask are read.
// A window with j < 0 or j + (steps - 1) s >= n_frames is not read and its sums are not written.  grid (B, S).
// kVec: 64x64 frames, 16-byte fp32 / 8-byte bf16 loads; otherwise scalar loads (see the grid section's header).
// ------------------------------------------------------------------------------------------------
namespace fno {

template <typename TFrame, bool kVec>
__global__ void __launch_bounds__(kMtThreads)
    window_metrics_kernel(const float* __restrict__ preds_seq, const TFrame* __restrict__ frames_in,
                          const TFrame* __restrict__ frames_out, const long long* __restrict__ starts, int batch,
                          int steps, int time_step_size, long long n_frames, int hw, float* __restrict__ out) {
  const int b = blockIdx.x, k = blockIdx.y;
  const long long j = starts[b];
  if (j < 0 || j + static_cast<long long>(steps - 1) * time_step_size >= n_frames) return;
  const size_t plane = static_cast<size_t>(k) * batch + b;
  const float* p = preds_seq + plane * 2 * hw;   // channel 0 = u
  const TFrame* l = frames_out + static_cast<size_t>(j + static_cast<long long>(k) * time_step_size) * 3 * hw;
  const TFrame* m = frames_in + (static_cast<size_t>(j) * 3 + 2) * hw;
  if constexpr (kVec) {
    reduce_plane_sums<4>(kHW / 4, [&](int i, float (&pp)[4], float (&ll)[4]) {
      const float4 pv = __ldg(reinterpret_cast<const float4*>(p) + i);
      const float4 lv = gather_ld4<TFrame>(l + 4 * i), mv = gather_ld4<TFrame>(m + 4 * i);
      pp[0] = pv.x * mv.x, pp[1] = pv.y * mv.y, pp[2] = pv.z * mv.z, pp[3] = pv.w * mv.w;
      ll[0] = lv.x * mv.x, ll[1] = lv.y * mv.y, ll[2] = lv.z * mv.z, ll[3] = lv.w * mv.w;
    }, out, plane);
  } else {
    reduce_plane_sums<1>(hw, [&](int i, float (&pp)[1], float (&ll)[1]) {
      const float mv = frame_ld(m + i);
      pp[0] = __ldg(p + i) * mv, ll[0] = frame_ld(l + i) * mv;
    }, out, plane);
  }
}

template <bool kVec>
static cudaError_t launch_window_metrics_impl(const float* preds_seq, const void* frames_in, const void* frames_out,
                                              const long long* starts, int steps, int batch, int time_step_size,
                                              long long n_frames, int frame_bf16, float* out, int hw, cudaStream_t stream) {
  dim3 grid(batch, steps);
  if (frame_bf16)
    window_metrics_kernel<__nv_bfloat16, kVec><<<grid, kMtThreads, 0, stream>>>(
        preds_seq, static_cast<const __nv_bfloat16*>(frames_in), static_cast<const __nv_bfloat16*>(frames_out), starts,
        batch, steps, time_step_size, n_frames, hw, out);
  else
    window_metrics_kernel<float, kVec><<<grid, kMtThreads, 0, stream>>>(
        preds_seq, static_cast<const float*>(frames_in), static_cast<const float*>(frames_out), starts, batch, steps,
        time_step_size, n_frames, hw, out);
  return cudaGetLastError();
}

cudaError_t launch_window_metrics(const float* preds_seq, const void* frames_in, const void* frames_out,
                                  const long long* starts, int steps, int batch, int time_step_size, long long n_frames,
                                  int frame_bf16, float* out, cudaStream_t stream) {
  return launch_window_metrics_impl<true>(preds_seq, frames_in, frames_out, starts, steps, batch, time_step_size, n_frames,
                                          frame_bf16, out, kHW, stream);
}
cudaError_t launch_grid_window_metrics(const float* preds_seq, const void* frames_in, const void* frames_out,
                                       const long long* starts, int steps, int batch, int time_step_size,
                                       long long n_frames, int frame_bf16, float* out, int h, int w, cudaStream_t stream) {
  return launch_window_metrics_impl<false>(preds_seq, frames_in, frames_out, starts, steps, batch, time_step_size,
                                           n_frames, frame_bf16, out, h * w, stream);
}

}  // namespace fno
