// The two non-network pieces of a training step (reference src/train_auto.py:233-260), each one launch:
//
//  * MseLoss (reference src/models/loss.py:22-37): mse = mean((p-l)^2), rmse = sqrt(mse), mae = mean|p-l|,
//    nmse = mse / mean(l^2) over the whole batch tensor.  The reference issues 5 reduction kernels; here one kernel
//    accumulates the three sums (fixed grid, fixed-order two-stage reduction: deterministic) and the last block to
//    finish turns them into the five scalars.  The backward kernel writes dL/dpreds for any combination of upstream
//    gradients of the four dict entries (the script calls loss["nmse"].backward()).
//  * torch.optim.Adam.step (train_auto.py:213,256; complex parameters as pairs of reals, no amsgrad): all parameter
//    tensors of the model in ONE launch through a pointer table, against ~10 multi-tensor launches of the reference.
//  * the per-step pieces of a graph-replayed training epoch (cfdbench_b200/train.py): index staging, Adam with its
//    coefficients read from a device table, and the loss log.
#include "fno_common.cuh"
#include "../../include/cfdbench_b200.h"

namespace fno {

// ------------------------------------------------------------------------------------------------ loss
constexpr int kLossThreads = 256;
constexpr int kLossBlocks = 296;  // 2 per SM; also the size of the partial-sum table

// One thread's share of the three sums sum (p-l)^2, sum |p-l|, sum l^2 over n elements, in loss_fwd_kernel's partition:
// float4 index i = block * kLossThreads + thread, grid-stride nblocks * kLossThreads, the n % 4 tail in block 0.  With
// `aligned` false the same four elements are read one by one (a slice of a [K][B][2][H][W] tensor at odd H*W is only
// 4-byte aligned), so the sums do not depend on the alignment.
__device__ __forceinline__ void loss_thread_sums(const float* __restrict__ preds, const float* __restrict__ labels, size_t n,
                                                 bool aligned, unsigned block, unsigned nblocks, float& se, float& sa,
                                                 float& sl) {
  const size_t n4 = n / 4;
  const float4* p4 = reinterpret_cast<const float4*>(preds);
  const float4* l4 = reinterpret_cast<const float4*>(labels);
  for (size_t i = static_cast<size_t>(block) * kLossThreads + threadIdx.x; i < n4;
       i += static_cast<size_t>(nblocks) * kLossThreads) {
    float4 p, l;
    if (aligned) {
      p = __ldg(p4 + i);
      l = __ldg(l4 + i);
    } else {
      p = make_float4(__ldg(preds + 4 * i), __ldg(preds + 4 * i + 1), __ldg(preds + 4 * i + 2), __ldg(preds + 4 * i + 3));
      l = make_float4(__ldg(labels + 4 * i), __ldg(labels + 4 * i + 1), __ldg(labels + 4 * i + 2), __ldg(labels + 4 * i + 3));
    }
    const float d[4] = {p.x - l.x, p.y - l.y, p.z - l.z, p.w - l.w};
    const float lv[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      se = fmaf(d[c], d[c], se);
      sa += fabsf(d[c]);
      sl = fmaf(lv[c], lv[c], sl);
    }
  }
  if (block == 0)  // tail (n not a multiple of 4)
    for (size_t i = n4 * 4 + threadIdx.x; i < n; i += kLossThreads) {
      const float d = preds[i] - labels[i];
      se = fmaf(d, d, se);
      sa += fabsf(d);
      sl = fmaf(labels[i], labels[i], sl);
    }
}

// The block's sums into partials[block][3]; the last of nblocks blocks to arrive (ticket) sums the table in a fixed
// order (double accumulation), writes out[0..4] = mse, rmse, mae, nmse, mean(l^2) and re-arms the ticket.  Returns true
// in thread 0 of that block, after its out[] stores.
__device__ __forceinline__ bool loss_block_reduce(float se, float sa, float sl, size_t n, unsigned block, unsigned nblocks,
                                                  float* __restrict__ partials, unsigned int* ticket,
                                                  float* __restrict__ out) {
  __shared__ float red[kLossThreads / 32][3];
  __shared__ bool last;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sa += __shfl_xor_sync(0xffffffffu, sa, o);
    sl += __shfl_xor_sync(0xffffffffu, sl, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    red[warp][0] = se;
    red[warp][1] = sa;
    red[warp][2] = sl;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int w = 0; w < kLossThreads / 32; ++w) {
      t[0] += red[w][0];
      t[1] += red[w][1];
      t[2] += red[w][2];
    }
    partials[block * 3 + 0] = t[0];
    partials[block * 3 + 1] = t[1];
    partials[block * 3 + 2] = t[2];
    __threadfence();
    last = atomicAdd(ticket, 1u) == nblocks - 1;
  }
  __syncthreads();
  if (last && threadIdx.x < 32) {  // one warp sums the table in a fixed order (double accumulation)
    __threadfence();
    double t[3] = {0.0, 0.0, 0.0};
    for (int b = threadIdx.x; b < static_cast<int>(nblocks); b += 32) {
      t[0] += static_cast<double>(partials[b * 3 + 0]);
      t[1] += static_cast<double>(partials[b * 3 + 1]);
      t[2] += static_cast<double>(partials[b * 3 + 2]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      t[0] += __shfl_xor_sync(0xffffffffu, t[0], o);
      t[1] += __shfl_xor_sync(0xffffffffu, t[1], o);
      t[2] += __shfl_xor_sync(0xffffffffu, t[2], o);
    }
    if (threadIdx.x == 0) {
      const double inv = 1.0 / static_cast<double>(n);
      const double mse = t[0] * inv, mae = t[1] * inv, ml2 = t[2] * inv;
      out[0] = static_cast<float>(mse);
      out[1] = static_cast<float>(sqrt(mse));
      out[2] = static_cast<float>(mae);
      out[3] = static_cast<float>(mse / ml2);
      out[4] = static_cast<float>(ml2);
      *ticket = 0u;  // ready for the next call on this scratch buffer
      return true;
    }
  }
  return false;
}

// out[0..4] = mse, rmse, mae, nmse, mean(l^2);  scratch: [kLossBlocks][3] floats + one uint32 ticket
__global__ void __launch_bounds__(kLossThreads)
    loss_fwd_kernel(const float* __restrict__ preds, const float* __restrict__ labels, size_t n, float* __restrict__ scratch,
                    float* __restrict__ out) {
  float se = 0.f, sa = 0.f, sl = 0.f;
  loss_thread_sums(preds, labels, n, true, blockIdx.x, gridDim.x, se, sa, sl);
  loss_block_reduce(se, sa, sl, n, blockIdx.x, gridDim.x, scratch,
                    reinterpret_cast<unsigned int*>(scratch + kLossBlocks * 3), out);
}

// dpreds = g_mse 2d/N + g_rmse d/(N rmse) + g_mae sign(d)/N + g_nmse 2d/(N mean(l^2))
__global__ void __launch_bounds__(kLossThreads)
    loss_bwd_kernel(const float* __restrict__ preds, const float* __restrict__ labels, const float* __restrict__ fwd,
                    const float* __restrict__ gout, float* __restrict__ dpreds, size_t n) {
  const float inv_n = 1.f / static_cast<float>(n);
  const float g_mse = gout[0], g_rmse = gout[1], g_mae = gout[2], g_nmse = gout[3];
  const float rmse = fwd[1], ml2 = fwd[4];
  const float kd = inv_n * (2.f * g_mse + (rmse > 0.f ? g_rmse / rmse : 0.f) + 2.f * g_nmse / ml2);
  const float ka = inv_n * g_mae;
  for (size_t i = static_cast<size_t>(blockIdx.x) * kLossThreads + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * kLossThreads) {
    const float d = preds[i] - labels[i];
    const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    dpreds[i] = fmaf(kd, d, ka * sgn);
  }
}

cudaError_t launch_loss_fwd(const float* preds, const float* labels, size_t n, float* scratch, float* out,
                            cudaStream_t stream) {
  loss_fwd_kernel<<<kLossBlocks, kLossThreads, 0, stream>>>(preds, labels, n, scratch, out);
  return cudaGetLastError();
}
cudaError_t launch_loss_bwd(const float* preds, const float* labels, const float* fwd, const float* gout, float* dpreds,
                            size_t n, cudaStream_t stream) {
  loss_bwd_kernel<<<kLossBlocks * 2, kLossThreads, 0, stream>>>(preds, labels, fwd, gout, dpreds, n);
  return cudaGetLastError();
}
size_t loss_scratch_bytes() { return (kLossBlocks * 3 + 4) * sizeof(float); }

// ------------------------------------------------------------------------------------------------ K-step loss
// The loss of a K-step rollout, (MseLoss(preds_0, labels_0) + ... + MseLoss(preds_{K-1}, labels_{K-1})) / K, in one launch
// each way.  Step k's slice is preds_seq + k n / labels_seq + k n (n = B*2*H*W), on grid row blockIdx.y = k with
// loss_fwd_kernel's block partition and reduction order, so row k of the output is bit-identical to fno_loss_fwd on that
// slice (on an aligned copy when the slice is not 16-byte aligned).  The quotient by K is a multiplication by the float32
// reciprocal 1/K: that is what `sum(...) / K` computes on 0-dim CUDA tensors (a CUDA tensor divided by a Python number),
// and what autograd's DivBackward computes for the upstream gradient.

// out[k][0..4] = fno_loss_fwd's five scalars of step k; out[steps][c] = (out[0][c] + ... + out[steps-1][c]) * (1/steps),
// summed left to right in float32.  scratch: [steps][kLossBlocks][3] floats, then steps + 1 uint32 tickets.
__global__ void __launch_bounds__(kLossThreads)
    loss_seq_fwd_kernel(const float* __restrict__ preds_seq, const float* __restrict__ labels_seq, size_t n, int steps,
                        float* __restrict__ scratch, float* __restrict__ out) {
  const int k = blockIdx.y;
  const float* preds = preds_seq + static_cast<size_t>(k) * n;
  const float* labels = labels_seq + static_cast<size_t>(k) * n;
  const bool aligned = ((reinterpret_cast<uintptr_t>(preds) | reinterpret_cast<uintptr_t>(labels)) & 15) == 0;
  unsigned int* tickets = reinterpret_cast<unsigned int*>(scratch + static_cast<size_t>(steps) * kLossBlocks * 3);
  float se = 0.f, sa = 0.f, sl = 0.f;
  loss_thread_sums(preds, labels, n, aligned, blockIdx.x, gridDim.x, se, sa, sl);
  if (!loss_block_reduce(se, sa, sl, n, blockIdx.x, gridDim.x, scratch + static_cast<size_t>(k) * kLossBlocks * 3,
                         tickets + k, out + static_cast<size_t>(k) * 5))
    return;
  // thread 0 of the block that finished step k: the last step to finish forms the aggregate row
  __threadfence();
  if (atomicAdd(tickets + steps, 1u) != static_cast<unsigned int>(steps) - 1) return;
  __threadfence();
  const float inv_k = 1.f / static_cast<float>(steps);
#pragma unroll
  for (int c = 0; c < 5; ++c) {
    float s = __ldcg(out + c);
    for (int j = 1; j < steps; ++j) s = s + __ldcg(out + static_cast<size_t>(j) * 5 + c);
    out[static_cast<size_t>(steps) * 5 + c] = s * inv_k;
  }
  tickets[steps] = 0u;
}

// dpreds_seq[k] = fno_loss_bwd(preds_k, labels_k, fwd[k], gout * (1/steps)): gout holds the upstream gradients of the
// aggregate row's (mse, rmse, mae, nmse).  loss_bwd_kernel's arithmetic, element by element (scalar accesses).
__global__ void __launch_bounds__(kLossThreads)
    loss_seq_bwd_kernel(const float* __restrict__ preds_seq, const float* __restrict__ labels_seq,
                        const float* __restrict__ fwd, const float* __restrict__ gout, float* __restrict__ dpreds_seq,
                        size_t n, int steps) {
  const int k = blockIdx.y;
  const size_t off = static_cast<size_t>(k) * n;
  const float inv_k = 1.f / static_cast<float>(steps);
  const float inv_n = 1.f / static_cast<float>(n);
  const float g_mse = gout[0] * inv_k, g_rmse = gout[1] * inv_k, g_mae = gout[2] * inv_k, g_nmse = gout[3] * inv_k;
  const float rmse = fwd[static_cast<size_t>(k) * 5 + 1], ml2 = fwd[static_cast<size_t>(k) * 5 + 4];
  const float kd = inv_n * (2.f * g_mse + (rmse > 0.f ? g_rmse / rmse : 0.f) + 2.f * g_nmse / ml2);
  const float ka = inv_n * g_mae;
  for (size_t i = static_cast<size_t>(blockIdx.x) * kLossThreads + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * kLossThreads) {
    const float d = preds_seq[off + i] - labels_seq[off + i];
    const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    dpreds_seq[off + i] = fmaf(kd, d, ka * sgn);
  }
}

cudaError_t launch_loss_seq_fwd(const float* preds_seq, const float* labels_seq, size_t n, int steps, float* scratch,
                                float* out, cudaStream_t stream) {
  loss_seq_fwd_kernel<<<dim3(kLossBlocks, steps), kLossThreads, 0, stream>>>(preds_seq, labels_seq, n, steps, scratch, out);
  return cudaGetLastError();
}
cudaError_t launch_loss_seq_bwd(const float* preds_seq, const float* labels_seq, const float* fwd, const float* gout,
                                float* dpreds_seq, size_t n, int steps, cudaStream_t stream) {
  loss_seq_bwd_kernel<<<dim3(kLossBlocks * 2, steps), kLossThreads, 0, stream>>>(preds_seq, labels_seq, fwd, gout,
                                                                                 dpreds_seq, n, steps);
  return cudaGetLastError();
}
size_t loss_seq_scratch_bytes(int steps) {
  return static_cast<size_t>(steps) * kLossBlocks * 3 * sizeof(float) + (static_cast<size_t>(steps) + 1) * 4;
}

// ------------------------------------------------------------------------------------------------ Adam
constexpr int kAdamThreads = 256;
constexpr int kAdamChunk = kAdamThreads * 4;  // elements per block

struct AdamArgs {
  fno_adam_tensors t;
  int first_block[FNO_ADAM_MAX_TENSORS + 1];  // prefix sum of ceil(n_i / kAdamChunk)
  float lr, beta1, beta2, eps, weight_decay, step_size, inv_bc2_sqrt;
  // kDevCoef: (step_size, inv_bc2_sqrt) = coef[*cursor], read on the device (a graph replays one launch for every step)
  const float2* coef;
  const int* cursor;
  int n_coef;
};

// The bias-corrected step size and 1/sqrt(bc2) of 1-based step `step`, as torch.optim.Adam forms them: in double, from
// lr, beta1 and beta2 as the float32 values the kernel sees.  The one copy of this arithmetic: launch_adam_step_ex and
// the device coefficient table (fno_adam_coefficients) both call it, so the two paths cannot drift apart.
void adam_coefficients(float lr, float beta1, float beta2, long long step, float* step_size, float* inv_bc2_sqrt) {
  const double bc1 = 1.0 - pow(static_cast<double>(beta1), static_cast<double>(step));
  const double bc2 = 1.0 - pow(static_cast<double>(beta2), static_cast<double>(step));
  *step_size = static_cast<float>(static_cast<double>(lr) / bc1);
  *inv_bc2_sqrt = static_cast<float>(1.0 / sqrt(bc2));
}

// The EMA decay of 1-based step `step`: min(decay, 1 - step^(-3/4)), in double, rounded to float32.  This is diffusers'
// EMAModel.get_decay(step) with use_ema_warmup=True, inv_gamma=1, power=3/4, update_after_step=0, min_decay=0 (its
// `step - 1` plus its `1 +`), so step 1 gives 0 and the EMA starts as a copy of the weights.  The one copy of this
// arithmetic: launch_adam_step_ex and the device table (fno_ema_decays) both call it.
float ema_decay_at(double decay, long long step) {
  const double warm = 1.0 - pow(static_cast<double>(step), -0.75);
  return static_cast<float>(warm < decay ? warm : decay);
}

// What the _ex Adam adds (all unused by adam_step_kernel): the clip coefficient (device, written by fno_grad_norm), the
// EMA tensors of the table's entries and the step's EMA decay (by value, or decay_tab[*cursor] with kDevCoef).
struct AdamExt {
  const float* clip;
  float* ema[FNO_ADAM_MAX_TENSORS];
  const float* decay_tab;
  float decay;
};

// torch.optim.Adam, single-tensor formulation (torch/optim/adam.py _single_tensor_adam):
//   g += wd p;  m = lerp(m, g, 1-b1);  v = b2 v + (1-b2) g g;  p -= step_size * m / (sqrt(v)/sqrt(bc2) + eps)
//   kDevCoef = false: step_size / inv_bc2_sqrt by value (fno_adam_step);  true: from coef[*cursor] (fno_adam_step_dev),
//   and a cursor outside 0..n_coef-1 makes the launch write nothing
//   kClip: g = g * clip coefficient before the weight decay (clip_grad_norm_ before optimizer.step());
//   kEma: ema = fmaf(-d, p_new - ema, p_new) with the step's decay d, p_new still in registers
template <bool kDevCoef, bool kClip, bool kEma>
__device__ __forceinline__ void adam_update(const AdamArgs& a, const AdamExt& x) {
  float step_size = a.step_size, inv_bc2_sqrt = a.inv_bc2_sqrt;
  float decay = 0.f;
  if constexpr (kEma) decay = x.decay;
  if constexpr (kDevCoef) {
    const int c = *a.cursor;
    if (c < 0 || c >= a.n_coef) return;
    const float2 k = a.coef[c];
    step_size = k.x;
    inv_bc2_sqrt = k.y;
    if constexpr (kEma) decay = x.decay_tab[c];
  }
  float coef = 1.f;
  if constexpr (kClip) coef = *x.clip;
  int ti = 0;
#pragma unroll 1
  while (ti + 1 < a.t.count && static_cast<int>(blockIdx.x) >= a.first_block[ti + 1]) ++ti;
  const long long n = a.t.n[ti];
  float* __restrict__ p = static_cast<float*>(a.t.param[ti]);
  const float* __restrict__ g = static_cast<const float*>(a.t.grad[ti]);
  float* __restrict__ m = static_cast<float*>(a.t.exp_avg[ti]);
  float* __restrict__ v = static_cast<float*>(a.t.exp_avg_sq[ti]);
  float* __restrict__ e = nullptr;
  if constexpr (kEma) e = x.ema[ti];
  const long long base = static_cast<long long>(blockIdx.x - a.first_block[ti]) * kAdamChunk;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const long long i = base + r * kAdamThreads + threadIdx.x;
    if (i < n) {
      float gi = g[i];
      if constexpr (kClip) gi = gi * coef;
      const float pi = p[i];
      if (a.weight_decay != 0.f) gi = fmaf(a.weight_decay, pi, gi);
      float mi = m[i], vi = v[i];
      mi = fmaf(gi - mi, 1.f - a.beta1, mi);
      vi = fmaf(1.f - a.beta2, gi * gi, vi * a.beta2);
      const float denom = sqrtf(vi) * inv_bc2_sqrt + a.eps;
      m[i] = mi;
      v[i] = vi;
      const float pn = pi - step_size * (mi / denom);
      p[i] = pn;
      if constexpr (kEma) e[i] = fmaf(-decay, pn - e[i], pn);
    }
  }
}

template <bool kDevCoef>
__global__ void __launch_bounds__(kAdamThreads) adam_step_kernel(const __grid_constant__ AdamArgs a) {
  adam_update<kDevCoef, false, false>(a, AdamExt{});
}

template <bool kDevCoef, bool kClip, bool kEma>
__global__ void __launch_bounds__(kAdamThreads)
    adam_step_ex_kernel(const __grid_constant__ AdamArgs a, const __grid_constant__ AdamExt x) {
  adam_update<kDevCoef, kClip, kEma>(a, x);
}

static int adam_blocks(const fno_adam_tensors* t, AdamArgs& a) {
  a.t = *t;
  int blocks = 0;
  for (int i = 0; i < t->count; ++i) {
    a.first_block[i] = blocks;
    blocks += static_cast<int>((t->n[i] + kAdamChunk - 1) / kAdamChunk);
  }
  a.first_block[t->count] = blocks;
  return blocks;
}

// Without a clip coefficient or EMA tensors this launches adam_step_kernel, the plain update of fno_adam_step[_dev].
template <bool kDevCoef>
static cudaError_t launch_adam_ex(const AdamArgs& a, const AdamExt& x, int blocks, cudaStream_t stream) {
  if (blocks == 0) return cudaSuccess;
  const bool clip = x.clip != nullptr, ema = x.ema[0] != nullptr;
  if (clip && ema)
    adam_step_ex_kernel<kDevCoef, true, true><<<blocks, kAdamThreads, 0, stream>>>(a, x);
  else if (clip)
    adam_step_ex_kernel<kDevCoef, true, false><<<blocks, kAdamThreads, 0, stream>>>(a, x);
  else if (ema)
    adam_step_ex_kernel<kDevCoef, false, true><<<blocks, kAdamThreads, 0, stream>>>(a, x);
  else
    adam_step_kernel<kDevCoef><<<blocks, kAdamThreads, 0, stream>>>(a);
  return cudaGetLastError();
}

static AdamExt adam_ext(const fno_adam_tensors* t, const float* clip_coef, void* const* ema) {
  AdamExt x = {};
  x.clip = clip_coef;
  if (ema)
    for (int i = 0; i < t->count; ++i) x.ema[i] = static_cast<float*>(ema[i]);
  return x;
}

cudaError_t launch_adam_step_ex(const fno_adam_tensors* t, float lr, float beta1, float beta2, float eps, float weight_decay,
                                long long step, const float* clip_coef, void* const* ema, double ema_decay,
                                cudaStream_t stream) {
  AdamArgs a = {};
  const int blocks = adam_blocks(t, a);
  a.lr = lr;
  a.beta1 = beta1;
  a.beta2 = beta2;
  a.eps = eps;
  a.weight_decay = weight_decay;
  adam_coefficients(lr, beta1, beta2, step, &a.step_size, &a.inv_bc2_sqrt);
  AdamExt x = adam_ext(t, clip_coef, ema);
  if (ema) x.decay = ema_decay_at(ema_decay, step);
  return launch_adam_ex<false>(a, x, blocks, stream);
}

cudaError_t launch_adam_step_dev_ex(const fno_adam_tensors* t, const float* coef, int n_coef, const int* cursor, float beta1,
                                    float beta2, float eps, float weight_decay, const float* clip_coef, void* const* ema,
                                    const float* ema_decay_tab, cudaStream_t stream) {
  AdamArgs a = {};
  const int blocks = adam_blocks(t, a);
  a.beta1 = beta1;
  a.beta2 = beta2;
  a.eps = eps;
  a.weight_decay = weight_decay;
  a.coef = reinterpret_cast<const float2*>(coef);
  a.cursor = cursor;
  a.n_coef = n_coef;
  AdamExt x = adam_ext(t, clip_coef, ema);
  x.decay_tab = ema_decay_tab;
  return launch_adam_ex<true>(a, x, blocks, stream);
}

// ------------------------------------------------------------------------------------------------ global gradient norm
// ||g||_2 over the gradients of up to FNO_GRAD_NORM_MAX_TABLES Adam tables, torch.nn.utils.clip_grad_norm_'s total norm,
// in one launch of a fixed kNormBlocks x kNormThreads grid.  Thread t of block b sums g*g in float64 over the elements
// i = (b * kNormThreads + t) + k * kNormBlocks * kNormThreads of every tensor in table order; the block reduces its
// threads in a fixed shuffle / warp order into partials[b], and the last block to arrive (an integer ticket) sums the
// kNormBlocks partials in a fixed order.  No float atomics: the result does not depend on the block schedule.
constexpr int kNormThreads = 256;
constexpr int kNormBlocks = 264;   // 2 per SM of an H100 SXM; fixed, so the reduction order is too
constexpr int kNormMaxTensors = FNO_GRAD_NORM_MAX_TABLES * FNO_ADAM_MAX_TENSORS;

struct NormArgs {
  const float* grad[kNormMaxTensors];
  long long n[kNormMaxTensors];
  int count;
  float max_norm;
  float* out;           // [2]: norm, coef
  double* partials;     // [kNormBlocks], then a uint32 ticket
  float* log;           // log[*cursor] = norm (optional)
  int n_log;
  const int* cursor;
};

__global__ void __launch_bounds__(kNormThreads) grad_norm_kernel(const __grid_constant__ NormArgs a) {
  __shared__ double red[kNormThreads / 32];
  __shared__ bool last;
  const long long stride = static_cast<long long>(kNormBlocks) * kNormThreads;
  const long long first = static_cast<long long>(blockIdx.x) * kNormThreads + threadIdx.x;
  double s = 0.0;
#pragma unroll 1
  for (int j = 0; j < a.count; ++j) {
    const float* __restrict__ g = a.grad[j];
    const long long n = a.n[j];
#pragma unroll 4
    for (long long i = first; i < n; i += stride) {
      const double v = static_cast<double>(__ldg(g + i));
      s = fma(v, v, s);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = s;
  __syncthreads();
  unsigned int* ticket = reinterpret_cast<unsigned int*>(a.partials + kNormBlocks);
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kNormThreads / 32; ++w) t += red[w];
    a.partials[blockIdx.x] = t;
    __threadfence();
    last = atomicAdd(ticket, 1u) == kNormBlocks - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x >= 32) return;
  __threadfence();
  double t = 0.0;
  for (int b = threadIdx.x; b < kNormBlocks; b += 32) t += __ldcg(a.partials + b);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (threadIdx.x != 0) return;
  // clip_grad_norm_'s coefficient in float32, max_norm / (norm + 1e-6) clamped to at most 1, as torch evaluates it: a
  // Python number over a tensor is reciprocal(tensor) * number.  A NaN norm gives NaN and an infinite one 0, as
  // torch.clamp(max=1) gives them.
  const float norm = static_cast<float>(sqrt(t));
  const float q = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), a.max_norm);
  a.out[0] = norm;
  a.out[1] = q > 1.f ? 1.f : q;
  if (a.log) {
    const int c = *a.cursor;
    if (c >= 0 && c < a.n_log) a.log[c] = norm;
  }
  *ticket = 0u;   // ready for the next call on this scratch buffer
}

cudaError_t launch_grad_norm(const fno_adam_tensors* tables, int n_tables, float max_norm, float* out, void* scratch,
                             float* log, int n_log, const int* cursor, cudaStream_t stream) {
  NormArgs a = {};
  for (int k = 0; k < n_tables; ++k)
    for (int i = 0; i < tables[k].count; ++i) {
      a.grad[a.count] = static_cast<const float*>(tables[k].grad[i]);
      a.n[a.count] = tables[k].n[i];
      ++a.count;
    }
  a.max_norm = max_norm;
  a.out = out;
  a.partials = static_cast<double*>(scratch);
  a.log = log;
  a.n_log = n_log;
  a.cursor = cursor;
  grad_norm_kernel<<<kNormBlocks, kNormThreads, 0, stream>>>(a);
  return cudaGetLastError();
}
size_t grad_norm_scratch_bytes() { return kNormBlocks * sizeof(double) + 16; }

// ------------------------------------------------------------------------------------------------ graph-replayed steps
// A CUDA graph of one training step is replayed once per step of an epoch; what changes from step to step lives on the
// device and is indexed by a step cursor: the step's sample indices (a slice of the epoch's permutation), Adam's
// coefficients (a table row) and the slot of the step's loss in the epoch's log.  Both kernels below refuse a cursor that
// would read or write past their table and then write nothing.

// idx_out[i] = perm[cursor * stride + i], i < batch
__global__ void __launch_bounds__(256) stage_indices_kernel(const long long* __restrict__ perm, long long n_perm, int stride,
                                                            int batch, const int* __restrict__ cursor,
                                                            long long* __restrict__ idx_out) {
  const int c = *cursor;
  const long long base = static_cast<long long>(c) * stride;
  if (c < 0 || base + batch > n_perm) return;
  for (int i = threadIdx.x; i < batch; i += blockDim.x) idx_out[i] = perm[base + i];
}

// log[cursor][0..4] = loss_out[0..4], then ++cursor
__global__ void log_step_kernel(const float* __restrict__ loss_out, float* __restrict__ log, int n_log, int* cursor) {
  const int c = *cursor;
  if (c < 0 || c >= n_log) return;
#pragma unroll
  for (int k = 0; k < 5; ++k) log[static_cast<size_t>(c) * 5 + k] = loss_out[k];
  *cursor = c + 1;
}

cudaError_t launch_stage_indices(const long long* perm, long long n_perm, int stride, int batch, const int* cursor,
                                 long long* idx_out, cudaStream_t stream) {
  stage_indices_kernel<<<1, 256, 0, stream>>>(perm, n_perm, stride, batch, cursor, idx_out);
  return cudaGetLastError();
}
cudaError_t launch_log_step(const float* loss_out, float* log, int n_log, int* cursor, cudaStream_t stream) {
  log_step_kernel<<<1, 1, 0, stream>>>(loss_out, log, n_log, cursor);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ input noise
// inputs[b][e] += (std * z) * mask[b][e mod HW] where mask != 0, e over the flattened (2, H, W) frame of sample b.  The
// normal z of element e = 4q + r is component r of Box-Muller on Philox4x32-10(counter = (q, j, step_lo, step_hi),
// key = (seed_lo, seed_hi)), j = idx[b]: a pure function of (seed, step, j, e), whatever the batch slot, the launch or the
// replay.  step = *step_base (+ *step_offset), read on the device so that a captured launch sees each replay's step.
// One thread per quad; the 64x64 path moves a quad as one float4 (it never straddles the two channels).
// Noise streams (input_noise_stream_kernel, the per-step noise of a rollout): stream k draws from counter.x = q + (k << 16)
// instead of q.  q < 2 * 128 * 128 / 4 = 2^13, so streams k < 2^16 never share a counter, and stream 0 is the counter above:
// the same noise as add_input_noise_kernel, bit for bit.
constexpr int kNoiseThreads = 256;

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const unsigned lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const unsigned lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// curand's uniform in (0, 1]: x 2^-32 + 2^-33 in float32
__device__ __forceinline__ float noise_uniform(unsigned x) {
  return __fadd_rn(__fmul_rn(__uint2float_rn(x), 2.3283064365386963e-10f), 1.1641532182693481e-10f);
}

__device__ __forceinline__ float4 noise_normals(unsigned long long seed, unsigned long long step, unsigned j, unsigned q) {
  const uint4 x = philox4x32_10(make_uint4(q, j, static_cast<unsigned>(step), static_cast<unsigned>(step >> 32)),
                                make_uint2(static_cast<unsigned>(seed), static_cast<unsigned>(seed >> 32)));
  const float r0 = sqrtf(-2.f * logf(noise_uniform(x.x))), t0 = 2.f * noise_uniform(x.y);
  const float r1 = sqrtf(-2.f * logf(noise_uniform(x.z))), t1 = 2.f * noise_uniform(x.w);
  return make_float4(r0 * cospif(t0), r0 * sinpif(t0), r1 * cospif(t1), r1 * sinpif(t1));
}

// The body of both noise kernels for sample b = blockIdx.y and quad q.  kInPlace (add_input_noise_kernel, out == in):
// only the cells where mask != 0 are written.  Otherwise (input_noise_stream_kernel) out = in + noise where mask != 0 and
// out = in elsewhere, so `out` is a whole frame; `out` may still equal `in`.
// kSelect (the teacher-forced feed of a rollout step): sample b's frame is alt's where flags[b] != 0, in's otherwise -- a
// choice of source, so the frame that is not chosen is never read and nothing of it (a NaN included) reaches out.
// !kNoise: out = that frame, bit for bit (no noise drawn; idx, step_base and mask are not read).
template <bool kVec, bool kInPlace, bool kSelect = false, bool kNoise = true>
__device__ __forceinline__ void input_noise(const float* in, float* out, const float* __restrict__ mask,
                                            const long long* __restrict__ idx, int hw, float std, unsigned long long seed,
                                            const long long* __restrict__ step_base, const int* __restrict__ step_offset,
                                            unsigned stream, const float* alt = nullptr,
                                            const unsigned char* __restrict__ flags = nullptr) {
  static_assert(!(kInPlace && kSelect), "the select writes a whole frame");
  const int b = blockIdx.y;
  const int n_el = 2 * hw;
  const unsigned q = blockIdx.x * kNoiseThreads + threadIdx.x;
  if (4 * q >= static_cast<unsigned>(n_el)) return;
  const float* src = in;
  if constexpr (kSelect) src = flags[b] != 0 ? alt : in;
  const float* x = src + static_cast<size_t>(b) * n_el;
  float* y = out + static_cast<size_t>(b) * n_el;
  if constexpr (!kNoise) {
    if constexpr (kVec) {
      *reinterpret_cast<float4*>(y + 4 * q) = *reinterpret_cast<const float4*>(x + 4 * q);
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (static_cast<int>(4 * q) + r < n_el) y[4 * q + r] = x[4 * q + r];
    }
    return;
  }
  const unsigned long long step =
      static_cast<unsigned long long>(*step_base) + (step_offset ? static_cast<long long>(*step_offset) : 0ll);
  const float4 z = noise_normals(seed, step, static_cast<unsigned>(idx[b]), q + (stream << 16));
  const float zs[4] = {z.x, z.y, z.z, z.w};
  const float* m = mask + static_cast<size_t>(b) * hw;
  if constexpr (kVec) {   // hw % 4 == 0 and 16-byte aligned slices: the quad lies in one channel
    const int e = 4 * q, cell = e < hw ? e : e - hw;
    const float4 mv = __ldg(reinterpret_cast<const float4*>(m + cell));
    const float4 xv = *reinterpret_cast<const float4*>(x + e);
    const float ms[4] = {mv.x, mv.y, mv.z, mv.w};
    const float x0[4] = {xv.x, xv.y, xv.z, xv.w};
    float xs[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) xs[r] = fmaf(std * zs[r], ms[r], x0[r]);
    if constexpr (kInPlace) {
      if (ms[0] != 0.f && ms[1] != 0.f && ms[2] != 0.f && ms[3] != 0.f) {
        *reinterpret_cast<float4*>(y + e) = make_float4(xs[0], xs[1], xs[2], xs[3]);
      } else {
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (ms[r] != 0.f) y[e + r] = xs[r];
      }
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r) xs[r] = ms[r] != 0.f ? xs[r] : x0[r];
      *reinterpret_cast<float4*>(y + e) = make_float4(xs[0], xs[1], xs[2], xs[3]);
    }
  } else {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int e = 4 * q + r;
      if (e < n_el) {
        const float mv = __ldg(m + (e < hw ? e : e - hw));
        if constexpr (kInPlace) {
          if (mv != 0.f) y[e] = fmaf(std * zs[r], mv, x[e]);
        } else {
          const float xv = x[e];
          y[e] = mv != 0.f ? fmaf(std * zs[r], mv, xv) : xv;
        }
      }
    }
  }
}

template <bool kVec>
__global__ void __launch_bounds__(kNoiseThreads)
    add_input_noise_kernel(float* __restrict__ inputs, const float* __restrict__ mask, const long long* __restrict__ idx,
                           int hw, float std, unsigned long long seed, const long long* __restrict__ step_base,
                           const int* __restrict__ step_offset) {
  input_noise<kVec, true>(inputs, inputs, mask, idx, hw, std, seed, step_base, step_offset, 0u);
}

// out = in + noise of stream `stream` (input_noise's out-of-place form; in == out is allowed).  kSelect / !kNoise: the
// teacher-forced feed (launch_teacher_feed): out = (flags[b] ? alt : in) [+ noise].
template <bool kVec, bool kSelect = false, bool kNoise = true>
__global__ void __launch_bounds__(kNoiseThreads)
    input_noise_stream_kernel(const float* in, float* out, const float* __restrict__ mask, const long long* __restrict__ idx,
                              int hw, float std, unsigned long long seed, const long long* __restrict__ step_base,
                              const int* __restrict__ step_offset, unsigned stream, const float* alt,
                              const unsigned char* __restrict__ flags) {
  input_noise<kVec, false, kSelect, kNoise>(in, out, mask, idx, hw, std, seed, step_base, step_offset, stream, alt, flags);
}

cudaError_t launch_add_input_noise(float* inputs, const float* mask, const long long* idx, int n, int h, int w, float std,
                                   unsigned long long seed, const long long* step_base, const int* step_offset,
                                   cudaStream_t stream) {
  const int hw = h * w, quads = (2 * hw + 3) / 4;
  const dim3 grid((quads + kNoiseThreads - 1) / kNoiseThreads, n);
  const bool vec = hw % 4 == 0 && ((reinterpret_cast<uintptr_t>(inputs) | reinterpret_cast<uintptr_t>(mask)) & 15) == 0;
  if (vec)
    add_input_noise_kernel<true><<<grid, kNoiseThreads, 0, stream>>>(inputs, mask, idx, hw, std, seed, step_base,
                                                                      step_offset);
  else
    add_input_noise_kernel<false><<<grid, kNoiseThreads, 0, stream>>>(inputs, mask, idx, hw, std, seed, step_base,
                                                                       step_offset);
  return cudaGetLastError();
}

cudaError_t launch_input_noise_stream(const float* in, float* out, const float* mask, const long long* idx, int n, int h,
                                      int w, float std, unsigned long long seed, const long long* step_base,
                                      const int* step_offset, int noise_stream, cudaStream_t stream) {
  const int hw = h * w, quads = (2 * hw + 3) / 4;
  const dim3 grid((quads + kNoiseThreads - 1) / kNoiseThreads, n);
  const bool vec = hw % 4 == 0 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) |
                                    reinterpret_cast<uintptr_t>(mask)) & 15) == 0;
  const unsigned k = static_cast<unsigned>(noise_stream);
  if (vec)
    input_noise_stream_kernel<true><<<grid, kNoiseThreads, 0, stream>>>(in, out, mask, idx, hw, std, seed, step_base,
                                                                         step_offset, k, nullptr, nullptr);
  else
    input_noise_stream_kernel<false><<<grid, kNoiseThreads, 0, stream>>>(in, out, mask, idx, hw, std, seed, step_base,
                                                                          step_offset, k, nullptr, nullptr);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ teacher forcing
// The feed of a teacher-forced rollout step: out[b] = (flags[b] ? teacher[b] : pred[b]), plus the noise of stream
// `noise_stream` where mask != 0 when `noise` is set (input_noise_stream_kernel's select forms).  One launch.
cudaError_t launch_teacher_feed(const float* pred, const float* teacher, const unsigned char* flags, float* out,
                                const float* mask, const long long* idx, int n, int h, int w, float std,
                                unsigned long long seed, const long long* step_base, const int* step_offset, int noise_stream,
                                bool noise, cudaStream_t stream) {
  const int hw = h * w, quads = (2 * hw + 3) / 4;
  const dim3 grid((quads + kNoiseThreads - 1) / kNoiseThreads, n);
  const bool vec = hw % 4 == 0 && ((reinterpret_cast<uintptr_t>(pred) | reinterpret_cast<uintptr_t>(teacher) |
                                    reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(mask)) & 15) == 0;
  const unsigned k = static_cast<unsigned>(noise_stream);
#define FNO_FEED(V, N)                                                                                                     \
  input_noise_stream_kernel<V, true, N><<<grid, kNoiseThreads, 0, stream>>>(pred, out, mask, idx, hw, std, seed, step_base, \
                                                                            step_offset, k, teacher, flags)
  if (noise) {
    if (vec) FNO_FEED(true, true);
    else FNO_FEED(false, true);
  } else {
    if (vec) FNO_FEED(true, false);
    else FNO_FEED(false, false);
  }
#undef FNO_FEED
  return cudaGetLastError();
}

// flags[s - 1][i] = (u <= *prob) for rollout steps s = 1 .. steps - 1 and samples i < batch, u = the uniform in (0, 1] of
// word x of Philox4x32-10(counter = (s, j, step_lo, step_hi), key = (seed_lo, seed_hi)), j = idx[i], step = *step_base
// (+ *step_offset): a pure function of (seed, step, j, s), whatever the batch slot.  p = 0 never sets a flag (u > 0) and
// p = 1 always does (u <= 1); p and the step are read on the device, so a captured launch sees each replay's.
constexpr int kFlagThreads = 256;

__global__ void __launch_bounds__(kFlagThreads)
    teacher_flags_kernel(const long long* __restrict__ idx, int batch, int n, const float* __restrict__ prob,
                         unsigned long long seed, const long long* __restrict__ step_base,
                         const int* __restrict__ step_offset, unsigned char* __restrict__ flags) {
  const int i = blockIdx.x * kFlagThreads + threadIdx.x;
  if (i >= n) return;
  const int s = i / batch + 1, b = i - (s - 1) * batch;
  const unsigned long long step =
      static_cast<unsigned long long>(*step_base) + (step_offset ? static_cast<long long>(*step_offset) : 0ll);
  const uint4 x = philox4x32_10(make_uint4(static_cast<unsigned>(s), static_cast<unsigned>(idx[b]),
                                           static_cast<unsigned>(step), static_cast<unsigned>(step >> 32)),
                                make_uint2(static_cast<unsigned>(seed), static_cast<unsigned>(seed >> 32)));
  flags[i] = noise_uniform(x.x) <= *prob ? 1 : 0;
}

cudaError_t launch_teacher_flags(const long long* idx, int batch, int steps, const float* prob, unsigned long long seed,
                                 const long long* step_base, const int* step_offset, unsigned char* flags,
                                 cudaStream_t stream) {
  const int n = (steps - 1) * batch;
  teacher_flags_kernel<<<(n + kFlagThreads - 1) / kFlagThreads, kFlagThreads, 0, stream>>>(idx, batch, n, prob, seed,
                                                                                           step_base, step_offset, flags);
  return cudaGetLastError();
}

}  // namespace fno
