// extern "C" surface of libcfdbench_b200.so (declared in include/cfdbench_b200.h).
#include <stdio.h>
#include <string.h>

#include "../../include/cfdbench_b200.h"
#include "fno_common.cuh"

namespace fno {
cudaError_t launch_dft_fwd(const void*, void*, int, float, float, cudaStream_t);
cudaError_t launch_mode_mix(const void*, const void*, void*, void*, int, cudaStream_t);
cudaError_t launch_block_fused(const void*, const void*, const float*, const float*, void*, int, cudaStream_t);
size_t ym_image_bytes(int);
cudaError_t launch_pack_spectral(const void*, const void*, void*, int, cudaStream_t);
cudaError_t launch_unpack_spectral(const void*, void*, void*, int, cudaStream_t);
cudaError_t launch_dft_fwd_tc(const void*, void*, int, float, float, cudaStream_t);
cudaError_t launch_pack_mix_operand(const void*, void*, cudaStream_t);
cudaError_t launch_pack_mix_operand_direct(const void*, const void*, void*, int, cudaStream_t);
size_t mix_operand_bytes();
cudaError_t launch_gather_batch(const void*, const void*, const float*, const int*, const long long*, int, int, int, float*,
                                float*, float*, float*, cudaStream_t);
cudaError_t launch_loss_fwd(const float*, const float*, size_t, float*, float*, cudaStream_t);
cudaError_t launch_loss_bwd(const float*, const float*, const float*, const float*, float*, size_t, cudaStream_t);
size_t loss_scratch_bytes();
void adam_coefficients(float, float, float, long long, float*, float*);
cudaError_t launch_adam_step_ex(const fno_adam_tensors*, float, float, float, float, float, long long, const float*,
                                void* const*, double, cudaStream_t);
cudaError_t launch_adam_step_dev_ex(const fno_adam_tensors*, const float*, int, const int*, float, float, float, float,
                                    const float*, void* const*, const float*, cudaStream_t);
float ema_decay_at(double, long long);
cudaError_t launch_grad_norm(const fno_adam_tensors*, int, float, float*, void*, float*, int, const int*, cudaStream_t);
size_t grad_norm_scratch_bytes();
cudaError_t launch_stage_indices(const long long*, long long, int, int, const int*, long long*, cudaStream_t);
cudaError_t launch_log_step(const float*, float*, int, int*, cudaStream_t);
cudaError_t launch_inv_kx(const void*, void*, int, float, float, cudaStream_t);
template <typename TAct>
cudaError_t launch_block_tc(int, const void*, const void*, const float*, const float*, void*, float*, const float*, int,
                            cudaStream_t);
template <typename TAct>
cudaError_t launch_lift(const float*, const float*, const float*, const float*, const float*, const float*,
                        const float*, void*, int, int, cudaStream_t);
template <typename TAct>
cudaError_t launch_project_tc(const void*, const float*, const float*, const float*, const float*, const float*,
                              float*, int, cudaStream_t);
int project_bwd_rows_max();
int project_bwd_row();
cudaError_t launch_reduce_partials(const float*, int, int, float*, int, float*, int, float*, int, int, cudaStream_t);
template <typename TAct>
cudaError_t launch_project_bwd_tc(const void*, const float*, const float*, const float*, const float*, const float*, const float*,
                                  float*, float*, float*, int*, int, cudaStream_t);
template <typename TP, typename TQ, int NJ, int NI>
cudaError_t launch_chan_outer(const void*, const void*, float*, int*, int, cudaStream_t);
cudaError_t launch_multistep_metrics(const float*, const float*, const float*, float*, int, int, cudaStream_t);
cudaError_t launch_spectral_wgrad(const void*, const void*, void*, int, cudaStream_t);
cudaError_t launch_lift_bwd(const float*, const float*, const float*, const float*, const float*, const float*,
                            float*, float*, float*, int, int, int, cudaStream_t);
cudaError_t launch_lift_bwd_data(const float*, const float*, float*, float*, const float*, int, int, int, cudaStream_t,
                                 const unsigned char*);
// grid-generic fp32 path (fno_grid.cu)
bool grid_ok(int, int);
void grid_tables_release(int);
cudaError_t launch_grid_lift(const float*, const float*, const float*, const float*, const float*, const float*,
                             const float*, float*, int, int, int, int, cudaStream_t);
cudaError_t launch_grid_dft(const float*, void*, int, int, int, float, float, cudaStream_t);
cudaError_t launch_grid_inv_kx(const void*, float*, int, int, int, float, float, cudaStream_t);
cudaError_t launch_grid_block_out(int, const float*, const float*, const float*, const float*, float*, float*, const float*,
                                  int, int, int, cudaStream_t);
cudaError_t launch_grid_project(const float*, const float*, const float*, const float*, const float*, const float*, float*,
                                int, int, cudaStream_t);
cudaError_t launch_grid_project_bwd(const float*, const float*, const float*, const float*, const float*, const float*,
                                    const float*, float*, float*, float*, int, int, cudaStream_t);
int grid_project_bwd_parts(int, int);
int grid_project_bwd_row();
template <int NJ, int NI>
cudaError_t launch_grid_chan_outer(const float*, const float*, float*, int*, int, int, cudaStream_t);
cudaError_t launch_grid_lift_bwd(const float*, const float*, const float*, const float*, const float*, const float*,
                                 const float*, float*, float*, float*, const float*, int, int, int, int, int, cudaStream_t,
                                 const unsigned char*);
int grid_lift_bwd_parts(int);
int grid_lift_bwd_row();
size_t grid_bwd_partials_floats();
size_t grid_partials_offset_co();
size_t grid_partials_offset_lb();
cudaError_t launch_grid_multistep_metrics(const float*, const float*, const float*, float*, int, int, int, int, cudaStream_t);
cudaError_t launch_grid_gather_batch(const void*, const void*, const float*, const int*, const long long*, int, int, int,
                                     float*, float*, float*, float*, int, int, cudaStream_t);
cudaError_t launch_eval_sums(const float*, const float*, const float*, const float*, float*, int, int, int, cudaStream_t);
// training through K-step rollouts (fno_metrics.cu, fno_train_step.cu)
cudaError_t launch_gather_window(const void*, const void*, const float*, const int*, const long long*, int, int, int, float*,
                                 float*, float*, float*, int, int, long long, float*, cudaStream_t);
cudaError_t launch_grid_gather_window(const void*, const void*, const float*, const int*, const long long*, int, int, int,
                                      float*, float*, float*, float*, int, int, long long, float*, int, int, cudaStream_t);
cudaError_t launch_loss_seq_fwd(const float*, const float*, size_t, int, float*, float*, cudaStream_t);
cudaError_t launch_loss_seq_bwd(const float*, const float*, const float*, const float*, float*, size_t, int, cudaStream_t);
size_t loss_seq_scratch_bytes(int);
// rollout metrics of a device-resident split's windows (fno_metrics.cu)
cudaError_t launch_window_metrics(const float*, const void*, const void*, const long long*, int, int, int, long long, int,
                                  float*, cudaStream_t);
cudaError_t launch_grid_window_metrics(const float*, const void*, const void*, const long long*, int, int, int, long long,
                                       int, float*, int, int, cudaStream_t);
cudaError_t launch_add_input_noise(float*, const float*, const long long*, int, int, int, float, unsigned long long,
                                   const long long*, const int*, cudaStream_t);
cudaError_t launch_input_noise_stream(const float*, float*, const float*, const long long*, int, int, int, float,
                                      unsigned long long, const long long*, const int*, int, cudaStream_t);
cudaError_t launch_teacher_feed(const float*, const float*, const unsigned char*, float*, const float*, const long long*, int,
                                int, int, float, unsigned long long, const long long*, const int*, int, bool, cudaStream_t);
cudaError_t launch_teacher_flags(const long long*, int, int, const float*, unsigned long long, const long long*, const int*,
                                 unsigned char*, cudaStream_t);
}  // namespace fno

using namespace fno;

namespace fno {
void block_tc_release(int);
void block_fused_release(int);
void dft_fwd_tc_release(int);
}  // namespace fno

static thread_local char g_err[512] = "";

static int fail(int code, const char* what, cudaError_t e = cudaSuccess) {
  if (e != cudaSuccess)
    snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  else
    snprintf(g_err, sizeof(g_err), "%s", what);
  return code;
}
#define FNO_CUDA(call, what)                         \
  do {                                               \
    cudaError_t _e = (call);                         \
    if (_e != cudaSuccess) return fail(kErrCuda, what, _e); \
  } while (0)
#define FNO_TRY(call)        \
  do {                       \
    int _r = (call);         \
    if (_r != kOk) return _r; \
  } while (0)

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }
static inline bool bad_dtype(int d) { return d != FNO_ACT_F32 && d != FNO_ACT_BF16; }

// Alignment of a caller device pointer, checked by every entry point before any device work: `bytes` is the widest access
// the entry point's kernels make through it -- 16 for float4 / uint4 loads and stores, TMA and bulk copies; 8 for
// float2 (complex64), int64 and four-bf16 (uint2) accesses; 4 or 2 for scalar fp32 / bf16 ones.  A misaligned vector
// access faults the device (and ends the CUDA context); this refuses the call instead, naming the argument.  NULL passes
// (the entry point's own null checks decide about it).
static int need_align(const char* what, const char* arg, const void* p, unsigned bytes) {
  if ((reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0) return kOk;
  char msg[192];
  snprintf(msg, sizeof(msg), "%s: %s must be %u-byte aligned", what, arg, bytes);
  return fail(kErrArg, msg);
}
#define FNO_ALIGN(what, p, bytes) FNO_TRY(need_align(what, #p, p, bytes))
static inline unsigned act_bytes(int act_dtype) { return act_dtype == FNO_ACT_BF16 ? 2u : 4u; }   // scalar activation
static inline unsigned frame_vec_bytes(int frame_dtype) { return frame_dtype == FNO_ACT_BF16 ? 8u : 16u; }   // 4 frames

// ------------------------------------------------------------------------ per-step noise of a rollout (fno_noise)
// Call step s of a rollout driver is fed x_s (the call's inputs, or the prediction of step s-1).  With a noise descriptor
// and stream k0 + s >= 1 it is fed fed[s] = x_s + the noise of that stream instead (stream 0, the start frame's noise, is
// the gather's); fed is [steps][batch][2][h][w] like preds_seq.  nz == NULL: the frame is x_s, as without noise.
static int noise_args(const char* what, const fno_noise* nz, const float* fed, int steps) {
  char msg[160];
  if (!nz || !fed || !nz->idx || !nz->step_base || !(nz->std >= 0.f) || !isfinite(nz->std) || nz->k0 < 0 ||
      static_cast<long long>(nz->k0) + steps > FNO_NOISE_STREAMS) {
    snprintf(msg, sizeof(msg), "%s: bad noise argument", what);
    return fail(kErrArg, msg);
  }
  return kOk;
}

// What the per-step forward of a *_noise forward driver would refuse (fno_[grid_]forward with saved == NULL,
// fno_[grid_]forward_train otherwise), checked before the driver's first launch: with k0 >= 1 the noise of step 0 runs
// before step 0's forward, and reads inputs and mask.  Same status codes as the forward: 3 for n_layers, else 1.
static int noise_forward_args(const char* what, const fno_weights* w, const float* inputs, const float* mask,
                              const float* case_params, const fno_train_saved* saved, const fno_workspace* ws, int batch,
                              bool grid, int act_dtype) {
  char msg[160];
  bool bad = !w || !inputs || !mask || !ws || batch <= 0 || (!grid && bad_dtype(act_dtype));
  if (!bad && saved) {
    bad = !ws->ym || !ws->z;
  } else if (!bad) {
    const bool fused = !grid && act_dtype == FNO_ACT_BF16 && ws->ym_img;   // the bf16 inference blocks need no ym / z
    bad = !ws->act[0] || !ws->act[1] || !ws->xm || (!fused && (!ws->ym || !ws->z));
  }
  if (!bad) bad = (w->n_case_params > 0 && !case_params) || (grid && (!w->gx || !w->gy));
  if (bad) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) {
    snprintf(msg, sizeof(msg), "%s: n_layers out of range", what);
    return fail(kErrUnsupported, msg);
  }
  if (saved) {
    bool ok = saved->act[0] != nullptr;
    for (int l = 0; l < w->n_layers; ++l) ok = ok && saved->act[l + 1] && saved->pre[l] && saved->xm[l];
    if (!ok) {
      snprintf(msg, sizeof(msg), "%s: null saved buffer", what);
      return fail(kErrArg, msg);
    }
  }
  return kOk;
}

static inline bool noisy_step(const fno_noise* nz, int s) { return nz && nz->k0 + s > 0; }

// ------------------------------------------------------------------------ teacher forcing of a rollout (fno_teacher)
// With a teacher descriptor every call step s >= 1 is fed fed[s] = (flags[s-1][b] ? frames[s-1][b] : x_s[b]), plus the
// noise of stream k0 + s with a noise descriptor, written by one launch; the backward sweep recomputes step s from fed[s]
// and hands dpreds[s-1] alone (not fc0^T dL/da0 + dpreds[s-1]) to prediction s-1 of a forced sample.  The backward reads
// only flags.
static int teacher_args(const char* what, const fno_teacher* tc, const float* fed, bool forward) {
  char msg[160];
  if (!tc || !fed || !tc->flags || (forward && !tc->frames)) {
    snprintf(msg, sizeof(msg), "%s: bad teacher argument", what);
    return fail(kErrArg, msg);
  }
  FNO_ALIGN(what, tc->frames, 4);   // float4 only where every frame of the feed is 16-byte aligned
  return kOk;
}

static inline bool fed_step(const fno_noise* nz, const fno_teacher* tc, int s) {
  return (tc && s > 0) || noisy_step(nz, s);
}

// The caller frames of a forward / rollout / backward driver: the 64x64 lift and its backward read inputs and mask as
// float4 (vec = 16); the grid kernels read every frame one float at a time (vec = 4).  case_params is read per float.
static int frames_align(const char* what, const float* inputs, const float* mask, const float* case_params, unsigned vec) {
  FNO_ALIGN(what, inputs, vec);
  FNO_ALIGN(what, mask, vec);
  FNO_ALIGN(what, case_params, 4);
  return kOk;
}

// x = the frame call step s is fed: x itself, or fed[s] written from it (one launch)
static int feed_step(const fno_noise* nz, const fno_teacher* tc, float* fed, const float* mask, int s, size_t frame, int batch,
                     int h, int wd, const float*& x, void* stream) {
  if (!fed_step(nz, tc, s)) return kOk;
  float* out = fed + static_cast<size_t>(s) * frame;
  if (tc && s > 0) {
    FNO_CUDA(launch_teacher_feed(x, tc->frames + static_cast<size_t>(s - 1) * frame, tc->flags + static_cast<size_t>(s - 1) * batch,
                                 out, mask, nz ? reinterpret_cast<const long long*>(nz->idx) : nullptr, batch, h, wd,
                                 nz ? nz->std : 0.f, nz ? nz->seed : 0ull,
                                 nz ? reinterpret_cast<const long long*>(nz->step_base) : nullptr,
                                 nz ? reinterpret_cast<const int*>(nz->step_offset) : nullptr, nz ? nz->k0 + s : 0, nz != nullptr,
                                 S(stream)),
             "input_noise_stream_kernel(teacher)");
    x = out;
    return kOk;
  }
  FNO_CUDA(launch_input_noise_stream(x, out, mask, reinterpret_cast<const long long*>(nz->idx), batch, h, wd, nz->std,
                                     nz->seed, reinterpret_cast<const long long*>(nz->step_base),
                                     reinterpret_cast<const int*>(nz->step_offset), nz->k0 + s, S(stream)),
           "input_noise_stream_kernel");
  x = out;
  return kOk;
}

// the frame the backward sweep's step s was fed: fed[s] for a noisy step, else the input or the previous prediction
static inline const float* fed_frame(const fno_noise* nz, const fno_teacher* tc, const float* fed, const float* inputs,
                                     const float* preds_seq, int s, size_t frame) {
  if (fed_step(nz, tc, s)) return fed + static_cast<size_t>(s) * frame;
  return s > 0 ? preds_seq + static_cast<size_t>(s - 1) * frame : inputs;
}

extern "C" {

int fno_version(void) { return FNO_ABI_VERSION; }

int fno_destroy(void) {
  int dev = 0;
  FNO_CUDA(cudaGetDevice(&dev), "cudaGetDevice");
  if (dev < 0 || dev >= 64) return fail(kErrArg, "fno_destroy: device index");
  FNO_CUDA(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
  block_tc_release(dev);
  block_fused_release(dev);
  dft_fwd_tc_release(dev);
  grid_tables_release(dev);
  return kOk;
}
const char* fno_last_error(void) { return g_err; }

size_t fno_act_bytes(int batch, int act_dtype) {
  return static_cast<size_t>(batch) * kC * kHW * (act_dtype == FNO_ACT_BF16 ? 2 : 4);
}
size_t fno_modes_bytes(int batch) { return static_cast<size_t>(batch) * kModes * kC * sizeof(float2); }
size_t fno_z_bytes(int batch) { return static_cast<size_t>(batch) * kH * 2 * kM2 * kC * sizeof(float); }
size_t fno_ym_image_bytes(int batch) { return ym_image_bytes(batch); }
size_t fno_bwd_partials_bytes(void) {
  return (static_cast<size_t>(296) * (kProj * kC + kProj) + static_cast<size_t>(project_bwd_rows_max()) * project_bwd_row() +
          static_cast<size_t>(16) * kC * (5 + kMaxCaseParams + 1)) * sizeof(float);
}

int fno_pack_spectral_weights(const void* w1, const void* w2, void* wk, int conj_transpose, void* stream) {
  if (!w1 || !w2 || !wk) return fail(kErrArg, "fno_pack_spectral_weights: null pointer");
  FNO_TRY(need_align("fno_pack_spectral_weights", "weights1", w1, 8));
  FNO_TRY(need_align("fno_pack_spectral_weights", "weights2", w2, 8));
  FNO_ALIGN("fno_pack_spectral_weights", wk, 8);
  FNO_CUDA(launch_pack_spectral(w1, w2, wk, conj_transpose, S(stream)), "pack_spectral_kernel");
  return kOk;
}

size_t fno_mix_operand_bytes(void) { return mix_operand_bytes(); }

int fno_pack_mix_operand(const void* wk, void* wop, void* stream) {
  if (!wk || !wop) return fail(kErrArg, "fno_pack_mix_operand: null pointer");
  FNO_ALIGN("fno_pack_mix_operand", wk, 8);
  FNO_ALIGN("fno_pack_mix_operand", wop, 4);
  FNO_CUDA(launch_pack_mix_operand(wk, wop, S(stream)), "pack_mix_operand_kernel");
  return kOk;
}

int fno_pack_mix_operand_from_weights(const void* w1, const void* w2, void* wop, int conj_transpose, void* stream) {
  if (!w1 || !w2 || !wop) return fail(kErrArg, "fno_pack_mix_operand_from_weights: null pointer");
  FNO_TRY(need_align("fno_pack_mix_operand_from_weights", "weights1", w1, 8));
  FNO_TRY(need_align("fno_pack_mix_operand_from_weights", "weights2", w2, 8));
  FNO_ALIGN("fno_pack_mix_operand_from_weights", wop, 16);
  FNO_CUDA(launch_pack_mix_operand_direct(w1, w2, wop, conj_transpose, S(stream)), "pack_mix_operand_direct_kernel");
  return kOk;
}

int fno_unpack_spectral_grads(const void* gwk, void* gw1, void* gw2, void* stream) {
  if (!gwk || !gw1 || !gw2) return fail(kErrArg, "fno_unpack_spectral_grads: null pointer");
  FNO_ALIGN("fno_unpack_spectral_grads", gwk, 8);
  FNO_ALIGN("fno_unpack_spectral_grads", gw1, 8);
  FNO_ALIGN("fno_unpack_spectral_grads", gw2, 8);
  FNO_CUDA(launch_unpack_spectral(gwk, gw1, gw2, 0, S(stream)), "unpack_spectral_kernel");
  return kOk;
}

int fno_lift_fwd(const float* inputs, const float* mask, const float* case_params, const fno_weights* w,
                 void* act_out, int batch, int act_dtype, void* stream) {
  if (!inputs || !mask || !w || !act_out || batch <= 0 || bad_dtype(act_dtype))
    return fail(kErrArg, "fno_lift_fwd: bad argument");
  if (w->n_case_params > 0 && !case_params) return fail(kErrArg, "fno_lift_fwd: case_params is null");
  FNO_ALIGN("fno_lift_fwd", inputs, 16);
  FNO_ALIGN("fno_lift_fwd", mask, 16);
  FNO_ALIGN("fno_lift_fwd", case_params, 4);
  FNO_ALIGN("fno_lift_fwd", act_out, 16);
  cudaError_t e = act_dtype == FNO_ACT_F32
                      ? launch_lift<float>(inputs, mask, case_params, w->fc0_w, w->fc0_b, w->gx, w->gy, act_out, batch,
                                           w->n_case_params, S(stream))
                      : launch_lift<__nv_bfloat16>(inputs, mask, case_params, w->fc0_w, w->fc0_b, w->gx, w->gy,
                                                   act_out, batch, w->n_case_params, S(stream));
  FNO_CUDA(e, "lift_kernel");
  return kOk;
}

int fno_spectral_dft_fwd(const void* act_in, void* xm, int batch, int act_dtype, float s0, float s1, void* stream) {
  if (!act_in || !xm || batch <= 0 || bad_dtype(act_dtype)) return fail(kErrArg, "fno_spectral_dft_fwd: bad argument");
  FNO_ALIGN("fno_spectral_dft_fwd", act_in, 16);
  FNO_ALIGN("fno_spectral_dft_fwd", xm, act_dtype == FNO_ACT_BF16 ? 16u : 8u);   // launch_dft_fwd_tc requires 16
  if (act_dtype == FNO_ACT_BF16) {   // bf16 planes: the two-GEMM tensor-core kernel (fno_dft_fwd_tc.cu)
    FNO_CUDA(launch_dft_fwd_tc(act_in, xm, batch, s0, s1, S(stream)), "dft_fwd_tc_kernel");
    return kOk;
  }
  FNO_CUDA(launch_dft_fwd(act_in, xm, batch, s0, s1, S(stream)), "dft_fwd_kernel");
  return kOk;
}

int fno_mode_mix(const void* xm, const void* wk, void* ym, int batch, void* stream) {
  if (!xm || !wk || !ym || batch <= 0) return fail(kErrArg, "fno_mode_mix: bad argument");
  FNO_ALIGN("fno_mode_mix", xm, 16);
  FNO_TRY(need_align("fno_mode_mix", "wop", wk, 16));
  FNO_ALIGN("fno_mode_mix", ym, 8);
  FNO_CUDA(launch_mode_mix(xm, wk, ym, nullptr, batch, S(stream)), "mode_mix_tc_kernel");
  return kOk;
}

int fno_mode_mix_image(const void* xm, const void* wk, void* ym_img, int batch, void* stream) {
  if (!xm || !wk || !ym_img || batch <= 0) return fail(kErrArg, "fno_mode_mix_image: bad argument");
  FNO_ALIGN("fno_mode_mix_image", xm, 16);
  FNO_TRY(need_align("fno_mode_mix_image", "wop", wk, 16));
  FNO_ALIGN("fno_mode_mix_image", ym_img, 4);
  FNO_CUDA(launch_mode_mix(xm, wk, nullptr, ym_img, batch, S(stream)), "mode_mix_tc_kernel(image)");
  return kOk;
}

int fno_block_fused(const void* ym_img, const void* act_in, const float* w0t, const float* bias, void* act_out, int batch,
                    void* stream) {
  if (!ym_img || !act_in || !w0t || !act_out || batch <= 0) return fail(kErrArg, "fno_block_fused: bad argument");
  FNO_ALIGN("fno_block_fused", ym_img, 16);
  FNO_TRY(need_align("fno_block_fused", "act_in_bf16", act_in, 16));
  FNO_ALIGN("fno_block_fused", w0t, 4);
  FNO_ALIGN("fno_block_fused", bias, 4);
  FNO_TRY(need_align("fno_block_fused", "act_out_bf16", act_out, 16));
  FNO_CUDA(launch_block_fused(ym_img, act_in, w0t, bias, act_out, batch, S(stream)), "block_fused_kernel");
  return kOk;
}

int fno_spectral_inv_kx(const void* ym, void* z, int batch, float s0, float s1, void* stream) {
  if (!ym || !z || batch <= 0) return fail(kErrArg, "fno_spectral_inv_kx: bad argument");
  FNO_ALIGN("fno_spectral_inv_kx", ym, 8);
  FNO_ALIGN("fno_spectral_inv_kx", z, 4);
  FNO_CUDA(launch_inv_kx(ym, z, batch, s0, s1, S(stream)), "inv_kx_kernel");
  return kOk;
}

int fno_block_out(int epilogue, const void* z, const void* act_in, const float* w0t, const float* bias, void* act_out,
                  float* pre_out, const float* pre_in, int batch, int act_dtype, void* stream) {
  if (!z || !act_in || !w0t || !act_out || batch <= 0 || bad_dtype(act_dtype))
    return fail(kErrArg, "fno_block_out: bad argument");
  if (epilogue == FNO_EPI_GELU_SAVE_PRE && !pre_out) return fail(kErrArg, "fno_block_out: pre_out is null");
  if (epilogue == FNO_EPI_MUL_DGELU && !pre_in) return fail(kErrArg, "fno_block_out: pre_in is null");
  FNO_ALIGN("fno_block_out", z, 4);
  FNO_ALIGN("fno_block_out", act_in, act_bytes(act_dtype));
  FNO_ALIGN("fno_block_out", w0t, 4);
  FNO_ALIGN("fno_block_out", bias, 4);
  FNO_ALIGN("fno_block_out", act_out, act_bytes(act_dtype));
  FNO_ALIGN("fno_block_out", pre_out, 4);
  FNO_ALIGN("fno_block_out", pre_in, 4);
  cudaError_t e = act_dtype == FNO_ACT_F32
                      ? launch_block_tc<float>(epilogue, z, act_in, w0t, bias, act_out, pre_out, pre_in, batch, S(stream))
                      : launch_block_tc<__nv_bfloat16>(epilogue, z, act_in, w0t, bias, act_out, pre_out, pre_in, batch,
                                                       S(stream));
  FNO_CUDA(e, "block_tc_kernel");
  return kOk;
}

int fno_block_fwd(const fno_weights* w, int layer, const void* act_in, void* act_out, float* pre_out,
                  const fno_workspace* ws, int batch, int act_dtype, void* stream) {
  if (!w || !ws || layer < 0 || layer >= w->n_layers) return fail(kErrArg, "fno_block_fwd: bad argument");
  const bool fused = act_dtype == FNO_ACT_BF16 && ws->ym_img && !pre_out;   // TMA reads and writes the activations
  FNO_ALIGN("fno_block_fwd", act_in, 16);
  FNO_ALIGN("fno_block_fwd", act_out, fused ? 16u : act_bytes(act_dtype));
  FNO_ALIGN("fno_block_fwd", pre_out, 4);
  FNO_TRY(fno_spectral_dft_fwd(act_in, ws->xm, batch, act_dtype, 1.f, 1.f, stream));
  if (fused) {   // inference, bf16 storage: fused output stage
    FNO_TRY(fno_mode_mix_image(ws->xm, w->spec_wk[layer], ws->ym_img, batch, stream));
    return fno_block_fused(ws->ym_img, act_in, w->w0t[layer], w->w0_b[layer], act_out, batch, stream);
  }
  FNO_TRY(fno_mode_mix(ws->xm, w->spec_wk[layer], ws->ym, batch, stream));
  const float inv = 1.f / static_cast<float>(kHW);
  FNO_TRY(fno_spectral_inv_kx(ws->ym, ws->z, batch, inv, 2.f * inv, stream));
  return fno_block_out(pre_out ? FNO_EPI_GELU_SAVE_PRE : FNO_EPI_GELU, ws->z, act_in, w->w0t[layer], w->w0_b[layer],
                       act_out, pre_out, nullptr, batch, act_dtype, stream);
}

int fno_project_fwd(const void* act_in, const float* mask, const fno_weights* w, float* preds, int batch,
                    int act_dtype, void* stream) {
  if (!act_in || !mask || !w || !preds || batch <= 0 || bad_dtype(act_dtype))
    return fail(kErrArg, "fno_project_fwd: bad argument");
  FNO_ALIGN("fno_project_fwd", act_in, act_bytes(act_dtype));
  FNO_ALIGN("fno_project_fwd", mask, 4);
  FNO_ALIGN("fno_project_fwd", preds, 4);
  cudaError_t e =
      act_dtype == FNO_ACT_F32
          ? launch_project_tc<float>(act_in, w->fc1_w, w->fc1_b, w->fc2_w, w->fc2_b, mask, preds, batch, S(stream))
          : launch_project_tc<__nv_bfloat16>(act_in, w->fc1_w, w->fc1_b, w->fc2_w, w->fc2_b, mask, preds, batch, S(stream));
  FNO_CUDA(e, "project_kernel");
  return kOk;
}

int fno_forward(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                float* preds, const fno_workspace* ws, int batch, int act_dtype, void* stream) {
  if (!w || !ws || !ws->act[0] || !ws->act[1] || !ws->xm) return fail(kErrArg, "fno_forward: bad workspace");
  if (!(act_dtype == FNO_ACT_BF16 && ws->ym_img) && (!ws->ym || !ws->z)) return fail(kErrArg, "fno_forward: bad workspace");
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) return fail(kErrUnsupported, "fno_forward: n_layers out of range");
  FNO_TRY(frames_align("fno_forward", inputs, mask, case_params, 16));
  FNO_ALIGN("fno_forward", preds, 4);
  FNO_TRY(fno_lift_fwd(inputs, mask, case_params, w, ws->act[0], batch, act_dtype, stream));
  int cur = 0;
  for (int l = 0; l < w->n_layers; ++l) {
    FNO_TRY(fno_block_fwd(w, l, ws->act[cur], ws->act[cur ^ 1], nullptr, ws, batch, act_dtype, stream));
    cur ^= 1;
  }
  return fno_project_fwd(ws->act[cur], mask, w, preds, batch, act_dtype, stream);
}

static int rollout_impl(const char* what, const fno_weights* w, const float* inputs, const float* mask,
                        const float* case_params, float* preds_seq, int steps, const fno_workspace* ws, const fno_noise* nz,
                        float* fed, int batch, int act_dtype, void* stream) {
  const fno_teacher* tc = nullptr;   // the inference rollout has no teacher
  char msg[160];
  if (steps < 0 || !preds_seq) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  FNO_TRY(frames_align(what, inputs, mask, case_params, 16));
  FNO_ALIGN(what, preds_seq, 16);   // step s + 1's lift reads preds_seq[s]
  FNO_ALIGN(what, fed, 16);
  const size_t frame = static_cast<size_t>(batch) * 2 * kHW;
  const float* cur = inputs;
  for (int s = 0; s < steps; ++s) {
    float* nxt = preds_seq + static_cast<size_t>(s) * frame;
    FNO_TRY(feed_step(nz, tc, fed, mask, s, frame, batch, kH, kW, cur, stream));
    FNO_TRY(fno_forward(w, cur, mask, case_params, nxt, ws, batch, act_dtype, stream));
    cur = nxt;
  }
  return kOk;
}

int fno_rollout(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                float* preds_seq, int steps, const fno_workspace* ws, int batch, int act_dtype, void* stream) {
  return rollout_impl("fno_rollout", w, inputs, mask, case_params, preds_seq, steps, ws, nullptr, nullptr, batch, act_dtype,
                      stream);
}

int fno_rollout_noise(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                      float* preds_seq, int steps, const fno_workspace* ws, const fno_noise* noise, float* fed, int batch,
                      int act_dtype, void* stream) {
  FNO_TRY(noise_args("fno_rollout_noise", noise, fed, steps));
  FNO_TRY(noise_forward_args("fno_rollout_noise", w, inputs, mask, case_params, nullptr, ws, batch, false, act_dtype));
  return rollout_impl("fno_rollout_noise", w, inputs, mask, case_params, preds_seq, steps, ws, noise, fed, batch, act_dtype,
                      stream);
}

size_t fno_rollout_host_scratch_bytes(int batch, int n_case_params, int steps) {
  const size_t b = static_cast<size_t>(batch);
  return (b * 2 * kHW + b * kHW + static_cast<size_t>(steps) * b * 2 * kHW) * sizeof(float) +
         ((b * n_case_params * sizeof(float) + 255) / 256) * 256;
}

int fno_rollout_host(const fno_weights* w, const float* inputs_host, const float* mask_host,
                     const float* case_params_host, float* preds_seq_host, int steps, const fno_workspace* ws,
                     void* dev_io, int batch, int act_dtype, void* stream) {
  if (!w || !inputs_host || !mask_host || !preds_seq_host || !dev_io || batch <= 0 || steps <= 0)
    return fail(kErrArg, "fno_rollout_host: bad argument");
  FNO_ALIGN("fno_rollout_host", dev_io, 16);   // the device frames it holds are the rollout's inputs / mask / preds_seq
  const size_t b = static_cast<size_t>(batch);
  float* d_in = static_cast<float*>(dev_io);
  float* d_mask = d_in + b * 2 * kHW;
  float* d_seq = d_mask + b * kHW;
  float* d_params = d_seq + static_cast<size_t>(steps) * b * 2 * kHW;
  cudaStream_t st = S(stream);
  FNO_CUDA(cudaMemcpyAsync(d_in, inputs_host, b * 2 * kHW * sizeof(float), cudaMemcpyHostToDevice, st), "H2D inputs");
  FNO_CUDA(cudaMemcpyAsync(d_mask, mask_host, b * kHW * sizeof(float), cudaMemcpyHostToDevice, st), "H2D mask");
  if (w->n_case_params > 0)
    FNO_CUDA(cudaMemcpyAsync(d_params, case_params_host, b * w->n_case_params * sizeof(float), cudaMemcpyHostToDevice, st),
             "H2D case_params");
  FNO_TRY(fno_rollout(w, d_in, d_mask, d_params, d_seq, steps, ws, batch, act_dtype, stream));
  FNO_CUDA(cudaMemcpyAsync(preds_seq_host, d_seq, static_cast<size_t>(steps) * b * 2 * kHW * sizeof(float),
                           cudaMemcpyDeviceToHost, st),
           "D2H preds");
  return kOk;
}

// fno_forward_train up to the saved set: the lift and the Fourier blocks, not the projection (the rollout backward
// recomputes a step's saved set with this; the projection's output is not part of it)
static int forward_train_body(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                              const fno_train_saved* saved, const fno_workspace* ws, int batch, int act_dtype, void* stream) {
  FNO_TRY(fno_lift_fwd(inputs, mask, case_params, w, saved->act[0], batch, act_dtype, stream));
  const float inv = 1.f / static_cast<float>(kHW);
  for (int l = 0; l < w->n_layers; ++l) {
    if (!saved->act[l + 1] || !saved->pre[l] || !saved->xm[l]) return fail(kErrArg, "fno_forward_train: null saved buffer");
    FNO_TRY(fno_spectral_dft_fwd(saved->act[l], saved->xm[l], batch, act_dtype, 1.f, 1.f, stream));
    FNO_TRY(fno_mode_mix(saved->xm[l], w->spec_wk[l], ws->ym, batch, stream));
    FNO_TRY(fno_spectral_inv_kx(ws->ym, ws->z, batch, inv, 2.f * inv, stream));
    FNO_TRY(fno_block_out(FNO_EPI_GELU_SAVE_PRE, ws->z, saved->act[l], w->w0t[l], w->w0_b[l], saved->act[l + 1],
                          saved->pre[l], nullptr, batch, act_dtype, stream));
  }
  return kOk;
}

int fno_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                      float* preds, const fno_train_saved* saved, const fno_workspace* ws, int batch,
                      int act_dtype, void* stream) {
  if (!w || !saved || !ws || !ws->ym || !ws->z) return fail(kErrArg, "fno_forward_train: bad argument");
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) return fail(kErrUnsupported, "fno_forward_train: n_layers");
  FNO_TRY(frames_align("fno_forward_train", inputs, mask, case_params, 16));
  FNO_ALIGN("fno_forward_train", preds, 4);
  FNO_TRY(forward_train_body(w, inputs, mask, case_params, saved, ws, batch, act_dtype, stream));
  return fno_project_fwd(saved->act[w->n_layers], mask, w, preds, batch, act_dtype, stream);
}

// The backward pass behind fno_backward and fno_backward_inputs.  g == NULL: no parameter gradients --
// every weight-gradient launch (the reduce_partials / chan_outer of fc1, fc2 and w0, spectral_wgrad,
// unpack_spectral_grads, lift_bwd) is skipped and only the data path runs.  d_inputs / d_case_params (either may be NULL)
// receive the lift's data adjoint of dL/da0 (lift_bwd_data_kernel); with both NULL and g set, the launches are exactly
// those of the parameter-only backward.
// The rollout backward's sweep runs it once per step with two modes the single-step entry points leave off:
//   accum    = 1: every parameter gradient is added to (the sweep's first step wrote it);
//   hand_off = 1: lift_bwd_data_kernel<true>: d_inputs = fc0[:, 0:2]^T dL/da0 + add (the next sweep step's upstream
//                 gradient when `add` is the previous prediction's; `add` alone for a sample whose `gate` is set),
//                 gradient when `add` is the previous prediction's), d_case_params += its share.
static int backward_impl(const char* what, const fno_weights* w, const fno_weights_bwd* wb, const float* inputs,
                         const float* mask, const float* case_params, const float* dpreds, const fno_train_saved* saved,
                         const fno_grads* g, const fno_bwd_scratch* sc, const fno_workspace* ws, int batch, int act_dtype,
                         void* stream, float* d_inputs, float* d_case_params, int accum = 0, int hand_off = 0,
                         const float* add = nullptr, const unsigned char* gate = nullptr) {
  char msg[128];
  if (!w || !wb || !inputs || !mask || !dpreds || !saved || !sc || !ws || batch <= 0 || bad_dtype(act_dtype)) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  if (!sc->d[0] || !sc->d[1] || !sc->dz1 || !sc->gm || !sc->gwk || !sc->partials || !ws->ym || !ws->z) {
    snprintf(msg, sizeof(msg), "%s: null scratch buffer", what);
    return fail(kErrArg, msg);
  }
  FNO_TRY(frames_align(what, inputs, mask, case_params, 16));
  FNO_ALIGN(what, dpreds, 4);   // read one float at a time by project_bwd_tc_kernel
  FNO_ALIGN(what, d_inputs, 16);
  FNO_ALIGN(what, d_case_params, 4);
  cudaStream_t st = S(stream);
  const int L = w->n_layers, p = w->n_case_params;
  const bool bf = act_dtype == FNO_ACT_BF16;
  // Small gradients: every CTA stores its share as one row of sc->partials and a second launch adds the rows up in index
  // order (reduce_partials_kernel) -- no atomics, so the gradients are bit-for-bit reproducible.  The targets accumulate
  // over batch chunks / launches: clear them first.
  float* part_co = sc->partials;                                   // chan_outer: up to 296 rows x (128*32 + 128)
  float* part_pb = part_co + static_cast<size_t>(296) * (kProj * kC + kProj);   // project_bwd: 16 * chunk rows x 386
  float* part_lb = part_pb + static_cast<size_t>(project_bwd_rows_max()) * project_bwd_row();   // lift_bwd
  // no memsets: every gradient is WRITTEN by its (first) reduction -- reduce_partials with accumulate = 0,
  // lift_bwd_reduce, unpack_spectral_grads -- and only further batch chunks of the project stage accumulate
  // ---- project backward (batch chunks bound the dz1 scratch) -> d[0] = dpre_{L-1}
  const size_t act_elt = bf ? 2 : 4;
  for (int b0 = 0; b0 < batch; b0 += FNO_BWD_CHUNK) {
    const int nb = (batch - b0 < FNO_BWD_CHUNK) ? batch - b0 : FNO_BWD_CHUNK;
    const char* a_l = static_cast<const char*>(saved->act[L]) + static_cast<size_t>(b0) * kC * kHW * act_elt;
    const float* pre = saved->pre[L - 1] + static_cast<size_t>(b0) * kC * kHW;
    float* dout = sc->d[0] + static_cast<size_t>(b0) * kC * kHW;
    const float* dp = dpreds + static_cast<size_t>(b0) * 2 * kHW;
    const float* mk = mask + static_cast<size_t>(b0) * kHW;
    int rows = 0;
    cudaError_t e =
        bf ? launch_project_bwd_tc<__nv_bfloat16>(a_l, dp, mk, pre, w->fc1_w, w->fc1_b, w->fc2_w, dout, sc->dz1, part_pb, &rows, nb, st)
           : launch_project_bwd_tc<float>(a_l, dp, mk, pre, w->fc1_w, w->fc1_b, w->fc2_w, dout, sc->dz1, part_pb, &rows, nb, st);
    FNO_CUDA(e, "project_bwd_tc_kernel");
    if (!g) continue;   // data-only: the partial rows just written are never reduced
    const int acc_c = (accum || b0 > 0) ? 1 : 0;
    FNO_CUDA(launch_reduce_partials(part_pb, rows, project_bwd_row(), g->fc2_w, 2 * kProj, g->fc1_b, kProj, g->fc2_b, 2, acc_c, st),
             "reduce(fc2.weight | fc1.bias | fc2.bias)");
    int n_co = 0;
    e = bf ? launch_chan_outer<float, __nv_bfloat16, 128, 32>(sc->dz1, a_l, part_co, &n_co, nb, st)
           : launch_chan_outer<float, float, 128, 32>(sc->dz1, a_l, part_co, &n_co, nb, st);
    FNO_CUDA(e, "chan_outer_kernel(fc1)");
    FNO_CUDA(launch_reduce_partials(part_co, n_co, kProj * kC + kProj, g->fc1_w, kProj * kC, nullptr, 0, nullptr, 0, acc_c, st),
             "reduce(fc1.weight)");
  }
  // ---- Fourier blocks, last to first
  const float inv = 1.f / static_cast<float>(kHW);
  int cur = 0;
  for (int l = L - 1; l >= 0; --l) {
    float* dpre = sc->d[cur];
    float* dnext = sc->d[cur ^ 1];
    if (g) {
      int n_co = 0;
      cudaError_t e = bf ? launch_chan_outer<float, __nv_bfloat16, 32, 32>(dpre, saved->act[l], part_co, &n_co, batch, st)
                         : launch_chan_outer<float, float, 32, 32>(dpre, saved->act[l], part_co, &n_co, batch, st);
      FNO_CUDA(e, "chan_outer_kernel(w0)");
      FNO_CUDA(launch_reduce_partials(part_co, n_co, kC * kC + kC, g->w0_w[l], kC * kC, g->w0_b[l], kC, nullptr, 0, accum, st),
               "reduce(w0.weight | w0.bias)");
    }
    FNO_TRY(fno_spectral_dft_fwd(dpre, sc->gm, batch, FNO_ACT_F32, inv, 2.f * inv, stream));
    if (g) {
      FNO_CUDA(launch_spectral_wgrad(saved->xm[l], sc->gm, sc->gwk, batch, st), "spectral_wgrad_kernel");
      FNO_CUDA(launch_unpack_spectral(sc->gwk, g->spec_w1[l], g->spec_w2[l], accum, st), "unpack_spectral_kernel");
    }
    FNO_TRY(fno_mode_mix(sc->gm, wb->spec_wkT[l], ws->ym, batch, stream));
    FNO_TRY(fno_spectral_inv_kx(ws->ym, ws->z, batch, 1.f, 1.f, stream));
    FNO_TRY(fno_block_out(l > 0 ? FNO_EPI_MUL_DGELU : FNO_EPI_PLAIN, ws->z, dpre, wb->w0[l], nullptr, dnext, nullptr,
                          l > 0 ? saved->pre[l - 1] : nullptr, batch, FNO_ACT_F32, stream));
    cur ^= 1;
  }
  // sc->d[cur] = dL/da0, the gradient at the lift output (a bf16-stored a0 is differentiated straight through)
  if (g)
    FNO_CUDA(launch_lift_bwd(sc->d[cur], inputs, mask, case_params, w->gx, w->gy, g->fc0_w, g->fc0_b, part_lb, batch, p, accum,
                             st),
             "lift_bwd_kernel");
  if (d_inputs || d_case_params)
    FNO_CUDA(launch_lift_bwd_data(sc->d[cur], w->fc0_w, d_inputs, d_case_params, hand_off ? add : nullptr, hand_off, batch, p, st,
                                  hand_off ? gate : nullptr),
             "lift_bwd_data_kernel");
  return kOk;
}

int fno_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                 const float* case_params, const float* dpreds, const fno_train_saved* saved,
                 const fno_grads* g, const fno_bwd_scratch* sc, const fno_workspace* ws, int batch,
                 int act_dtype, void* stream) {
  if (!g) return fail(kErrArg, "fno_backward: bad argument");
  return backward_impl("fno_backward", w, wb, inputs, mask, case_params, dpreds, saved, g, sc, ws, batch, act_dtype, stream,
                       nullptr, nullptr);
}

int fno_backward_inputs(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                        const float* case_params, const float* dpreds, const fno_train_saved* saved,
                        const fno_grads* grads, const fno_bwd_scratch* scratch, const fno_workspace* ws,
                        float* d_inputs, float* d_case_params, int batch, int act_dtype, void* stream) {
  if (w && (w->n_case_params < 0 || w->n_case_params > kMaxCaseParams))
    return fail(kErrArg, "fno_backward_inputs: n_case_params out of range");
  if (w && w->n_case_params == 0) d_case_params = nullptr;   // nothing to write
  if (!grads && !d_inputs && !d_case_params) return fail(kErrArg, "fno_backward_inputs: no output requested");
  return backward_impl("fno_backward_inputs", w, wb, inputs, mask, case_params, dpreds, saved, grads, scratch, ws, batch,
                       act_dtype, stream, d_inputs, d_case_params);
}

// The arguments of the batch and window gathers: the 64x64 kernels (vec) move four frame elements at a time -- float4, or
// uint2 for bf16 frames -- and store float4; the grid kernels move one element at a time.
static int gather_align(const char* what, const void* frames_in, const void* frames_out, const float* case_table,
                        const int32_t* case_ids, const int64_t* idx, int frame_dtype, const float* inputs, const float* label,
                        const float* mask, const float* case_params, const float* labels_seq, bool vec) {
  const unsigned f = vec ? frame_vec_bytes(frame_dtype) : (frame_dtype == FNO_ACT_BF16 ? 2u : 4u), o = vec ? 16u : 4u;
  FNO_ALIGN(what, frames_in, f);
  FNO_ALIGN(what, frames_out, f);
  FNO_ALIGN(what, case_table, 4);
  FNO_ALIGN(what, case_ids, 4);
  FNO_ALIGN(what, idx, 8);
  FNO_ALIGN(what, inputs, o);
  FNO_ALIGN(what, label, o);
  FNO_ALIGN(what, mask, o);
  FNO_ALIGN(what, case_params, 4);
  FNO_ALIGN(what, labels_seq, o);
  return kOk;
}

// ------------------------------------------------------------------------ training through a rollout (64x64 and grids)
// Checks shared by the rollout training entry points: everything is validated before any device work.
static int rollout_bwd_args(const char* what, const fno_weights* w, const fno_weights_bwd* wb, const float* inputs,
                            const float* mask, const float* preds_seq, const float* dpreds_seq, int steps,
                            const fno_train_saved* saved, const fno_grads* g, const fno_bwd_scratch* sc, const fno_workspace* ws,
                            const float* carry, const float* d_inputs, const float* d_case_params, int batch) {
  char msg[160];
  if (steps < 1 || !w || !wb || !inputs || !mask || !dpreds_seq || !saved || !sc || !ws || batch <= 0 ||
      (steps > 1 && (!preds_seq || !carry))) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) {
    snprintf(msg, sizeof(msg), "%s: n_layers out of range", what);
    return fail(kErrUnsupported, msg);
  }
  if (w->n_case_params < 0 || w->n_case_params > kMaxCaseParams) {
    snprintf(msg, sizeof(msg), "%s: n_case_params out of range", what);
    return fail(kErrArg, msg);
  }
  if (!g && !d_inputs && !d_case_params) {
    snprintf(msg, sizeof(msg), "%s: no output requested", what);
    return fail(kErrArg, msg);
  }
  if (!sc->d[0] || !sc->d[1] || !sc->dz1 || !sc->gm || !sc->gwk || !sc->partials || !ws->ym || !ws->z) {
    snprintf(msg, sizeof(msg), "%s: null scratch buffer", what);
    return fail(kErrArg, msg);
  }
  if ((carry && carry == d_inputs) || (carry && carry == dpreds_seq)) {
    snprintf(msg, sizeof(msg), "%s: carry must be a buffer of its own", what);
    return fail(kErrArg, msg);
  }
  return kOk;
}

static int rollout_forward_train_impl(const char* what, const fno_weights* w, const float* inputs, const float* mask,
                                      const float* case_params, float* preds_seq, int steps, const fno_train_saved* saved,
                                      const fno_workspace* ws, const fno_noise* nz, const fno_teacher* tc, float* fed,
                                      int batch, int act_dtype, void* stream) {
  char msg[160];
  if (steps < 1 || !inputs || !preds_seq || batch <= 0) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  FNO_TRY(frames_align(what, inputs, mask, case_params, 16));
  FNO_ALIGN(what, preds_seq, 16);   // step s + 1's lift reads preds_seq[s]
  FNO_ALIGN(what, fed, 16);
  const size_t frame = static_cast<size_t>(batch) * 2 * kHW;
  const float* cur = inputs;
  for (int s = 0; s < steps; ++s) {
    float* nxt = preds_seq + static_cast<size_t>(s) * frame;
    FNO_TRY(feed_step(nz, tc, fed, mask, s, frame, batch, kH, kW, cur, stream));
    FNO_TRY(fno_forward_train(w, cur, mask, case_params, nxt, saved, ws, batch, act_dtype, stream));
    cur = nxt;
  }
  return kOk;
}

int fno_rollout_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                              float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws, int batch,
                              int act_dtype, void* stream) {
  return rollout_forward_train_impl("fno_rollout_forward_train", w, inputs, mask, case_params, preds_seq, steps, saved, ws,
                                    nullptr, nullptr, nullptr, batch, act_dtype, stream);
}

int fno_rollout_forward_train_noise(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                    float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws,
                                    const fno_noise* noise, float* fed, int batch, int act_dtype, void* stream) {
  FNO_TRY(noise_args("fno_rollout_forward_train_noise", noise, fed, steps));
  FNO_TRY(noise_forward_args("fno_rollout_forward_train_noise", w, inputs, mask, case_params, saved, ws, batch, false,
                             act_dtype));
  return rollout_forward_train_impl("fno_rollout_forward_train_noise", w, inputs, mask, case_params, preds_seq, steps, saved,
                                    ws, noise, nullptr, fed, batch, act_dtype, stream);
}

int fno_rollout_forward_train_feed(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                   float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws,
                                   const fno_noise* noise, const fno_teacher* teacher, float* fed, int batch, int act_dtype,
                                   void* stream) {
  const char* what = "fno_rollout_forward_train_feed";
  if (noise) FNO_TRY(noise_args(what, noise, fed, steps));
  FNO_TRY(teacher_args(what, teacher, fed, true));
  FNO_TRY(noise_forward_args(what, w, inputs, mask, case_params, saved, ws, batch, false, act_dtype));
  return rollout_forward_train_impl(what, w, inputs, mask, case_params, preds_seq, steps, saved, ws, noise, teacher, fed, batch,
                                    act_dtype, stream);
}

static int rollout_backward_impl(const char* what, const fno_weights* w, const fno_weights_bwd* wb, const float* inputs,
                                 const float* mask, const float* case_params, const float* preds_seq, const float* dpreds_seq,
                                 int steps, const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                                 const fno_workspace* ws, const fno_noise* nz, const fno_teacher* tc, const float* fed,
                                 float* carry, float* d_inputs, float* d_case_params, int batch, int act_dtype, void* stream) {
  char msg[160];
  if (w && w->n_case_params == 0) d_case_params = nullptr;   // nothing to write
  FNO_TRY(rollout_bwd_args(what, w, wb, inputs, mask, preds_seq, dpreds_seq, steps, saved, grads, scratch, ws, carry, d_inputs,
                           d_case_params, batch));
  if (bad_dtype(act_dtype)) {
    snprintf(msg, sizeof(msg), "%s: bad act_dtype", what);
    return fail(kErrArg, msg);
  }
  // the sweep's recomputed lift and lift backward read its frames (inputs, preds_seq, fed) as float4; its hand-off
  // writes carry / d_inputs and reads dpreds_seq as float4
  FNO_TRY(frames_align(what, inputs, mask, case_params, 16));
  FNO_ALIGN(what, preds_seq, 16);
  FNO_ALIGN(what, dpreds_seq, 16);
  FNO_ALIGN(what, fed, 16);
  FNO_ALIGN(what, carry, 16);
  FNO_ALIGN(what, d_inputs, 16);
  FNO_ALIGN(what, d_case_params, 4);
  const size_t frame = static_cast<size_t>(batch) * 2 * kHW;
  if (d_case_params)   // every sweep step adds its share
    FNO_CUDA(cudaMemsetAsync(d_case_params, 0, static_cast<size_t>(batch) * w->n_case_params * sizeof(float), S(stream)),
             "memset(d_case_params)");
  for (int s = steps - 1; s >= 0; --s) {
    const float* x = fed_frame(nz, tc, fed, inputs, preds_seq, s, frame);
    FNO_TRY(forward_train_body(w, x, mask, case_params, saved, ws, batch, act_dtype, stream));
    const float* up = s == steps - 1 ? dpreds_seq + static_cast<size_t>(s) * frame : carry;
    FNO_TRY(backward_impl(what, w, wb, x, mask, case_params, up, saved, grads, scratch, ws, batch, act_dtype, stream,
                          s > 0 ? carry : d_inputs, d_case_params, s != steps - 1 ? 1 : 0, 1,
                          s > 0 ? dpreds_seq + static_cast<size_t>(s - 1) * frame : nullptr,
                          tc && s > 0 ? tc->flags + static_cast<size_t>(s - 1) * batch : nullptr));
  }
  return kOk;
}

int fno_rollout_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                         const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                         const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                         const fno_workspace* ws, float* carry, float* d_inputs, float* d_case_params, int batch, int act_dtype,
                         void* stream) {
  return rollout_backward_impl("fno_rollout_backward", w, wb, inputs, mask, case_params, preds_seq, dpreds_seq, steps, saved,
                               grads, scratch, ws, nullptr, nullptr, nullptr, carry, d_inputs, d_case_params, batch, act_dtype,
                               stream);
}

int fno_rollout_backward_noise(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                               const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                               const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                               const fno_workspace* ws, const fno_noise* noise, const float* fed, float* carry,
                               float* d_inputs, float* d_case_params, int batch, int act_dtype, void* stream) {
  FNO_TRY(noise_args("fno_rollout_backward_noise", noise, fed, steps));
  return rollout_backward_impl("fno_rollout_backward_noise", w, wb, inputs, mask, case_params, preds_seq, dpreds_seq, steps,
                               saved, grads, scratch, ws, noise, nullptr, fed, carry, d_inputs, d_case_params, batch, act_dtype,
                               stream);
}

int fno_rollout_backward_feed(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                              const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                              const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                              const fno_workspace* ws, const fno_noise* noise, const fno_teacher* teacher, const float* fed,
                              float* carry, float* d_inputs, float* d_case_params, int batch, int act_dtype, void* stream) {
  const char* what = "fno_rollout_backward_feed";
  if (noise) FNO_TRY(noise_args(what, noise, fed, steps));
  FNO_TRY(teacher_args(what, teacher, fed, false));
  return rollout_backward_impl(what, w, wb, inputs, mask, case_params, preds_seq, dpreds_seq, steps, saved, grads, scratch, ws,
                               noise, teacher, fed, carry, d_inputs, d_case_params, batch, act_dtype, stream);
}

int fno_multistep_metrics(const float* preds_seq, const float* label_u, const float* mask, float* sums, int steps,
                          int batch, void* stream) {
  if (!preds_seq || !label_u || !mask || !sums || steps <= 0 || batch <= 0)
    return fail(kErrArg, "fno_multistep_metrics: bad argument");
  FNO_ALIGN("fno_multistep_metrics", preds_seq, 16);
  FNO_ALIGN("fno_multistep_metrics", label_u, 16);
  FNO_ALIGN("fno_multistep_metrics", mask, 16);
  FNO_ALIGN("fno_multistep_metrics", sums, 4);
  FNO_CUDA(launch_multistep_metrics(preds_seq, label_u, mask, sums, steps, batch, S(stream)), "multistep_metrics_kernel");
  return kOk;
}

int fno_gather_batch(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                     const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                     float* mask, float* case_params, void* stream) {
  if (!frames_in || !frames_out || !case_ids || !idx || !inputs || !label || !mask || n_idx <= 0 || n_case_params < 0 ||
      n_case_params > kMaxCaseParams || bad_dtype(frame_dtype) || (n_case_params > 0 && (!case_table || !case_params)))
    return fail(kErrArg, "fno_gather_batch: bad argument");
  FNO_TRY(gather_align("fno_gather_batch", frames_in, frames_out, case_table, case_ids, idx, frame_dtype, inputs, label, mask,
                       case_params, nullptr, true));
  FNO_CUDA(launch_gather_batch(frames_in, frames_out, case_table, reinterpret_cast<const int*>(case_ids),
                               reinterpret_cast<const long long*>(idx), n_idx, n_case_params, frame_dtype == FNO_ACT_BF16,
                               inputs, label, mask, case_params, S(stream)),
           "gather_batch_kernel");
  return kOk;
}

size_t fno_loss_scratch_bytes(void) { return loss_scratch_bytes(); }

int fno_loss_fwd(const float* preds, const float* labels, size_t n, void* scratch, float* out, void* stream) {
  if (!preds || !labels || !scratch || !out || n == 0) return fail(kErrArg, "fno_loss_fwd: bad argument");
  FNO_ALIGN("fno_loss_fwd", preds, 16);
  FNO_ALIGN("fno_loss_fwd", labels, 16);
  FNO_ALIGN("fno_loss_fwd", scratch, 4);
  FNO_ALIGN("fno_loss_fwd", out, 4);
  FNO_CUDA(launch_loss_fwd(preds, labels, n, static_cast<float*>(scratch), out, S(stream)), "loss_fwd_kernel");
  return kOk;
}

int fno_loss_bwd(const float* preds, const float* labels, const float* fwd, const float* gout, float* dpreds, size_t n,
                 void* stream) {
  if (!preds || !labels || !fwd || !gout || !dpreds || n == 0) return fail(kErrArg, "fno_loss_bwd: bad argument");
  FNO_ALIGN("fno_loss_bwd", preds, 4);
  FNO_ALIGN("fno_loss_bwd", labels, 4);
  FNO_ALIGN("fno_loss_bwd", fwd, 4);
  FNO_ALIGN("fno_loss_bwd", gout, 4);
  FNO_ALIGN("fno_loss_bwd", dpreds, 4);
  FNO_CUDA(launch_loss_bwd(preds, labels, fwd, gout, dpreds, n, S(stream)), "loss_bwd_kernel");
  return kOk;
}

static int adam_tensors_ok(const fno_adam_tensors* t) {
  if (!t || t->count < 0 || t->count > FNO_ADAM_MAX_TENSORS) return 0;
  for (int i = 0; i < t->count; ++i)
    if (!t->param[i] || !t->grad[i] || !t->exp_avg[i] || !t->exp_avg_sq[i] || t->n[i] <= 0) return 0;
  return 1;
}
static bool ema_ok(const fno_adam_tensors* t, void* const* ema) {
  if (!ema) return true;
  for (int i = 0; i < t->count; ++i)
    if (!ema[i]) return false;
  return true;
}
static inline bool decay_ok(double d) { return d >= 0.0 && d < 1.0; }   // false for NaN

// The checks and launch behind fno_adam_step and fno_adam_step_ex (clip_coef and ema NULL: the plain update); `what` is
// the entry point, named in fno_last_error().
static int adam_step_impl(const char* what, const fno_adam_tensors* t, float lr, float beta1, float beta2, float eps,
                          float weight_decay, int64_t step, const float* clip_coef, void* const* ema, double ema_decay,
                          void* stream) {
  const bool args_ok = step >= 1 && (!ema || decay_ok(ema_decay));
  if (!args_ok || !adam_tensors_ok(t) || !ema_ok(t, ema)) {
    char msg[96];
    snprintf(msg, sizeof(msg), "%s: %s", what, args_ok ? "bad tensor table" : "bad argument");
    return fail(kErrArg, msg);
  }
  FNO_ALIGN(what, clip_coef, 4);
  FNO_CUDA(launch_adam_step_ex(t, lr, beta1, beta2, eps, weight_decay, step, clip_coef, ema, ema_decay, S(stream)), what);
  return kOk;
}

// The same for fno_adam_step_dev and fno_adam_step_dev_ex.
static int adam_step_dev_impl(const char* what, const fno_adam_tensors* t, const float* coef, int n_coef,
                              const int32_t* cursor, float beta1, float beta2, float eps, float weight_decay,
                              const float* clip_coef, void* const* ema, const float* ema_decay_tab, void* stream) {
  const bool args_ok = coef && cursor && n_coef > 0 && (!ema || ema_decay_tab);
  if (!args_ok || !adam_tensors_ok(t) || !ema_ok(t, ema)) {
    char msg[96];
    snprintf(msg, sizeof(msg), "%s: %s", what, args_ok ? "bad tensor table" : "bad argument");
    return fail(kErrArg, msg);
  }
  FNO_ALIGN(what, coef, 8);   // one float2 per step
  FNO_ALIGN(what, cursor, 4);
  FNO_ALIGN(what, clip_coef, 4);
  FNO_ALIGN(what, ema_decay_tab, 4);
  FNO_CUDA(launch_adam_step_dev_ex(t, coef, n_coef, reinterpret_cast<const int*>(cursor), beta1, beta2, eps, weight_decay,
                                   clip_coef, ema, ema ? ema_decay_tab : nullptr, S(stream)),
           what);
  return kOk;
}

int fno_adam_step(const fno_adam_tensors* t, float lr, float beta1, float beta2, float eps, float weight_decay,
                  int64_t step, void* stream) {
  return adam_step_impl("fno_adam_step", t, lr, beta1, beta2, eps, weight_decay, step, nullptr, nullptr, 0.0, stream);
}

int fno_adam_step_dev(const fno_adam_tensors* t, const float* coef, int n_coef, const int32_t* cursor, float beta1,
                      float beta2, float eps, float weight_decay, void* stream) {
  return adam_step_dev_impl("fno_adam_step_dev", t, coef, n_coef, cursor, beta1, beta2, eps, weight_decay, nullptr, nullptr,
                            nullptr, stream);
}

int fno_adam_coefficients(float lr, float beta1, float beta2, int64_t first_step, int n, float* host_out) {
  if (!host_out || n <= 0 || first_step < 1) return fail(kErrArg, "fno_adam_coefficients: bad argument");
  for (int i = 0; i < n; ++i) adam_coefficients(lr, beta1, beta2, first_step + i, host_out + 2 * i, host_out + 2 * i + 1);
  return kOk;
}

// ---------------------------------------------------------------- gradient-norm clipping and the EMA of the weights
size_t fno_grad_norm_scratch_bytes(void) { return grad_norm_scratch_bytes(); }

int fno_grad_norm(const fno_adam_tensors* tables, int n_tables, float max_norm, float* out, void* scratch, float* log,
                  int n_log, const int32_t* cursor, void* stream) {
  if (!tables || n_tables < 1 || n_tables > FNO_GRAD_NORM_MAX_TABLES || !(max_norm > 0.f) || !isfinite(max_norm) || !out ||
      !scratch || (log && (!cursor || n_log <= 0)))
    return fail(kErrArg, "fno_grad_norm: bad argument");
  FNO_ALIGN("fno_grad_norm", out, 4);
  FNO_ALIGN("fno_grad_norm", scratch, 8);   // float64 partial sums
  FNO_ALIGN("fno_grad_norm", log, 4);
  FNO_ALIGN("fno_grad_norm", cursor, 4);
  for (int k = 0; k < n_tables; ++k) {   // only the grad and n fields are read
    const fno_adam_tensors& t = tables[k];
    if (t.count < 0 || t.count > FNO_ADAM_MAX_TENSORS) return fail(kErrArg, "fno_grad_norm: bad tensor table");
    for (int i = 0; i < t.count; ++i)
      if (!t.grad[i] || t.n[i] <= 0) return fail(kErrArg, "fno_grad_norm: bad tensor table");
  }
  FNO_CUDA(launch_grad_norm(tables, n_tables, max_norm, out, scratch, log, n_log, reinterpret_cast<const int*>(cursor),
                            S(stream)),
           "grad_norm_kernel");
  return kOk;
}

int fno_adam_step_ex(const fno_adam_tensors* t, float lr, float beta1, float beta2, float eps, float weight_decay,
                     int64_t step, const float* clip_coef, void* const* ema, double ema_decay, void* stream) {
  return adam_step_impl("fno_adam_step_ex", t, lr, beta1, beta2, eps, weight_decay, step, clip_coef, ema, ema_decay,
                        stream);
}

int fno_adam_step_dev_ex(const fno_adam_tensors* t, const float* coef, int n_coef, const int32_t* cursor, float beta1,
                         float beta2, float eps, float weight_decay, const float* clip_coef, void* const* ema,
                         const float* ema_decay_tab, void* stream) {
  return adam_step_dev_impl("fno_adam_step_dev_ex", t, coef, n_coef, cursor, beta1, beta2, eps, weight_decay, clip_coef, ema,
                            ema_decay_tab, stream);
}

int fno_ema_decays(double ema_decay, int64_t first_step, int n, float* host_out) {
  if (!host_out || n <= 0 || first_step < 1 || !decay_ok(ema_decay)) return fail(kErrArg, "fno_ema_decays: bad argument");
  for (int i = 0; i < n; ++i) host_out[i] = ema_decay_at(ema_decay, first_step + i);
  return kOk;
}

int fno_train_stage_indices(const int64_t* perm, int64_t n_perm, int stride, int batch, const int32_t* cursor,
                            int64_t* idx_out, void* stream) {
  if (!perm || !cursor || !idx_out || n_perm <= 0 || stride <= 0 || batch <= 0 || batch > stride || batch > n_perm)
    return fail(kErrArg, "fno_train_stage_indices: bad argument");
  FNO_ALIGN("fno_train_stage_indices", perm, 8);
  FNO_ALIGN("fno_train_stage_indices", cursor, 4);
  FNO_ALIGN("fno_train_stage_indices", idx_out, 8);
  FNO_CUDA(launch_stage_indices(reinterpret_cast<const long long*>(perm), n_perm, stride, batch,
                                reinterpret_cast<const int*>(cursor), reinterpret_cast<long long*>(idx_out), S(stream)),
           "stage_indices_kernel");
  return kOk;
}

int fno_train_log_step(const float* loss_out, float* log, int n_log, int32_t* cursor, void* stream) {
  if (!loss_out || !log || !cursor || n_log <= 0) return fail(kErrArg, "fno_train_log_step: bad argument");
  FNO_ALIGN("fno_train_log_step", loss_out, 4);
  FNO_ALIGN("fno_train_log_step", log, 4);
  FNO_ALIGN("fno_train_log_step", cursor, 4);
  FNO_CUDA(launch_log_step(loss_out, log, n_log, reinterpret_cast<int*>(cursor), S(stream)), "log_step_kernel");
  return kOk;
}

// ------------------------------------------------------------------------------------------------ K-step rollout training
static constexpr int kMaxSeqSteps = (65535 - 5) / 2;   // the gathers put 5 + 2 steps planes, the losses steps, on grid.y

static int gather_window_args(const char* what, const void* frames_in, const void* frames_out, const float* case_table,
                              const int32_t* case_ids, const int64_t* idx, int n_idx, int n_case_params, int frame_dtype,
                              const float* inputs, const float* mask, const float* case_params, int steps,
                              int time_step_size, int64_t n_frames, const float* labels_seq) {
  char msg[160];
  if (!frames_in || !frames_out || !case_ids || !idx || !inputs || !mask || !labels_seq || n_idx <= 0 ||
      n_case_params < 0 || n_case_params > kMaxCaseParams || bad_dtype(frame_dtype) ||
      (n_case_params > 0 && (!case_table || !case_params)) || steps < 1 || steps > kMaxSeqSteps || time_step_size < 1 ||
      n_frames < 1) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  return kOk;
}

int fno_gather_window(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                      const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                      float* mask, float* case_params, int steps, int time_step_size, int64_t n_frames, float* labels_seq,
                      void* stream) {
  FNO_TRY(gather_window_args("fno_gather_window", frames_in, frames_out, case_table, case_ids, idx, n_idx, n_case_params,
                             frame_dtype, inputs, mask, case_params, steps, time_step_size, n_frames, labels_seq));
  FNO_TRY(gather_align("fno_gather_window", frames_in, frames_out, case_table, case_ids, idx, frame_dtype, inputs, label, mask,
                       case_params, labels_seq, true));
  FNO_CUDA(launch_gather_window(frames_in, frames_out, case_table, reinterpret_cast<const int*>(case_ids),
                                reinterpret_cast<const long long*>(idx), n_idx, n_case_params, frame_dtype == FNO_ACT_BF16,
                                inputs, label, mask, case_params, steps, time_step_size, n_frames, labels_seq, S(stream)),
           "gather_window_kernel");
  return kOk;
}

size_t fno_loss_seq_scratch_bytes(int steps) { return steps < 1 ? 0 : loss_seq_scratch_bytes(steps); }

int fno_loss_seq_fwd(const float* preds_seq, const float* labels_seq, size_t n, int steps, void* scratch, float* out,
                     void* stream) {
  if (!preds_seq || !labels_seq || !scratch || !out || n == 0 || steps < 1 || steps > kMaxSeqSteps)
    return fail(kErrArg, "fno_loss_seq_fwd: bad argument");
  FNO_ALIGN("fno_loss_seq_fwd", preds_seq, 4);
  FNO_ALIGN("fno_loss_seq_fwd", labels_seq, 4);
  FNO_ALIGN("fno_loss_seq_fwd", scratch, 4);
  FNO_ALIGN("fno_loss_seq_fwd", out, 4);
  FNO_CUDA(launch_loss_seq_fwd(preds_seq, labels_seq, n, steps, static_cast<float*>(scratch), out, S(stream)),
           "loss_seq_fwd_kernel");
  return kOk;
}

int fno_loss_seq_bwd(const float* preds_seq, const float* labels_seq, const float* fwd, const float* gout, float* dpreds_seq,
                     size_t n, int steps, void* stream) {
  if (!preds_seq || !labels_seq || !fwd || !gout || !dpreds_seq || n == 0 || steps < 1 || steps > kMaxSeqSteps)
    return fail(kErrArg, "fno_loss_seq_bwd: bad argument");
  FNO_ALIGN("fno_loss_seq_bwd", preds_seq, 4);
  FNO_ALIGN("fno_loss_seq_bwd", labels_seq, 4);
  FNO_ALIGN("fno_loss_seq_bwd", fwd, 4);
  FNO_ALIGN("fno_loss_seq_bwd", gout, 4);
  FNO_ALIGN("fno_loss_seq_bwd", dpreds_seq, 4);
  FNO_CUDA(launch_loss_seq_bwd(preds_seq, labels_seq, fwd, gout, dpreds_seq, n, steps, S(stream)), "loss_seq_bwd_kernel");
  return kOk;
}

// ------------------------------------------------------------------------------------------------ grid-generic fp32 path
static int grid_arg(const char* what, int h, int w) {
  char msg[160];
  if (!grid_ok(h, w)) {
    snprintf(msg, sizeof(msg), "%s: grid %dx%d outside the supported range 24..128 x 24..128", what, h, w);
    return fail(kErrUnsupported, msg);
  }
  return kOk;
}

size_t fno_grid_act_bytes(int batch, int h, int w) {
  return static_cast<size_t>(batch) * kC * h * w * sizeof(float);
}
size_t fno_grid_z_bytes(int batch, int h) { return static_cast<size_t>(batch) * h * 2 * kM2 * kC * sizeof(float); }
size_t fno_grid_bwd_partials_bytes(int h, int w) {
  (void)h;
  (void)w;   // the partial rows come from a fixed number of CTAs: the size does not depend on the grid
  return grid_bwd_partials_floats() * sizeof(float);
}

int fno_grid_lift_fwd(const float* inputs, const float* mask, const float* case_params, const fno_weights* w,
                      float* act_out, int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_lift_fwd", h, wd));
  if (!inputs || !mask || !w || !act_out || batch <= 0 || !w->gx || !w->gy) return fail(kErrArg, "fno_grid_lift_fwd: bad argument");
  if (w->n_case_params > 0 && !case_params) return fail(kErrArg, "fno_grid_lift_fwd: case_params is null");
  FNO_ALIGN("fno_grid_lift_fwd", inputs, 4);
  FNO_ALIGN("fno_grid_lift_fwd", mask, 4);
  FNO_ALIGN("fno_grid_lift_fwd", case_params, 4);
  FNO_ALIGN("fno_grid_lift_fwd", act_out, 4);
  FNO_CUDA(launch_grid_lift(inputs, mask, case_params, w->fc0_w, w->fc0_b, w->gx, w->gy, act_out, batch, w->n_case_params, h,
                            wd, S(stream)),
           "grid_lift_kernel");
  return kOk;
}

int fno_grid_spectral_dft_fwd(const float* act_in, void* xm, int batch, int h, int wd, float s0, float s1, void* stream) {
  FNO_TRY(grid_arg("fno_grid_spectral_dft_fwd", h, wd));
  if (!act_in || !xm || batch <= 0) return fail(kErrArg, "fno_grid_spectral_dft_fwd: bad argument");
  FNO_ALIGN("fno_grid_spectral_dft_fwd", act_in, 4);
  FNO_ALIGN("fno_grid_spectral_dft_fwd", xm, 8);
  FNO_CUDA(launch_grid_dft(act_in, xm, batch, h, wd, s0, s1, S(stream)), "grid_dft_kernel");
  return kOk;
}

int fno_grid_spectral_inv_kx(const void* ym, float* z, int batch, int h, int wd, float s0, float s1, void* stream) {
  FNO_TRY(grid_arg("fno_grid_spectral_inv_kx", h, wd));
  if (!ym || !z || batch <= 0) return fail(kErrArg, "fno_grid_spectral_inv_kx: bad argument");
  FNO_ALIGN("fno_grid_spectral_inv_kx", ym, 8);
  FNO_ALIGN("fno_grid_spectral_inv_kx", z, 4);
  FNO_CUDA(launch_grid_inv_kx(ym, z, batch, h, wd, s0, s1, S(stream)), "grid_inv_kx_kernel");
  return kOk;
}

int fno_grid_block_out(int epilogue, const float* z, const float* act_in, const float* w0t, const float* bias, float* act_out,
                       float* pre_out, const float* pre_in, int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_block_out", h, wd));
  if (!z || !act_in || !w0t || !act_out || batch <= 0 || epilogue < FNO_EPI_GELU || epilogue > FNO_EPI_PLAIN)
    return fail(kErrArg, "fno_grid_block_out: bad argument");
  if (epilogue == FNO_EPI_GELU_SAVE_PRE && !pre_out) return fail(kErrArg, "fno_grid_block_out: pre_out is null");
  if (epilogue == FNO_EPI_MUL_DGELU && !pre_in) return fail(kErrArg, "fno_grid_block_out: pre_in is null");
  FNO_ALIGN("fno_grid_block_out", z, 16);
  FNO_ALIGN("fno_grid_block_out", act_in, 4);
  FNO_ALIGN("fno_grid_block_out", w0t, 4);
  FNO_ALIGN("fno_grid_block_out", bias, 4);
  FNO_ALIGN("fno_grid_block_out", act_out, 4);
  FNO_ALIGN("fno_grid_block_out", pre_out, 4);
  FNO_ALIGN("fno_grid_block_out", pre_in, 4);
  FNO_CUDA(launch_grid_block_out(epilogue, z, act_in, w0t, bias, act_out, pre_out, pre_in, batch, h, wd, S(stream)),
           "grid_block_out_kernel");
  return kOk;
}

int fno_grid_project_fwd(const float* act_in, const float* mask, const fno_weights* w, float* preds, int batch, int h, int wd,
                         void* stream) {
  FNO_TRY(grid_arg("fno_grid_project_fwd", h, wd));
  if (!act_in || !mask || !w || !preds || batch <= 0) return fail(kErrArg, "fno_grid_project_fwd: bad argument");
  FNO_ALIGN("fno_grid_project_fwd", act_in, 4);
  FNO_ALIGN("fno_grid_project_fwd", mask, 4);
  FNO_ALIGN("fno_grid_project_fwd", preds, 4);
  FNO_CUDA(launch_grid_project(act_in, w->fc1_w, w->fc1_b, w->fc2_w, w->fc2_b, mask, preds, batch, h * wd, S(stream)),
           "grid_project_kernel");
  return kOk;
}

// project backward over batch chunks of FNO_BWD_CHUNK (dz1 holds one chunk); gradients written when g_fc1_w is set
// (added to with accum = 1)
static int grid_project_bwd_impl(const float* act, const float* dpreds, const float* mask, const float* pre,
                                 const fno_weights* w, float* dpre_out, float* dz1, float* partials, float* g_fc1_w,
                                 float* g_fc1_b, float* g_fc2_w, float* g_fc2_b, int batch, int h, int wd, cudaStream_t st,
                                 int accum = 0) {
  const int hw = h * wd;
  float* part_pb = partials;
  float* part_co = partials + grid_partials_offset_co();
  const bool grads = g_fc1_w != nullptr;
  for (int b0 = 0; b0 < batch; b0 += FNO_BWD_CHUNK) {
    const int nb = (batch - b0 < FNO_BWD_CHUNK) ? batch - b0 : FNO_BWD_CHUNK;
    const size_t act_off = static_cast<size_t>(b0) * kC * hw;
    FNO_CUDA(launch_grid_project_bwd(act + act_off, dpreds + static_cast<size_t>(b0) * 2 * hw, mask + static_cast<size_t>(b0) * hw,
                                     pre + act_off, w->fc1_w, w->fc1_b, w->fc2_w, dpre_out + act_off, dz1,
                                     grads ? part_pb : nullptr, nb, hw, st),
             "grid_project_bwd_kernel");
    if (!grads) continue;
    const int acc_c = (accum || b0 > 0) ? 1 : 0;
    FNO_CUDA(launch_reduce_partials(part_pb, grid_project_bwd_parts(nb, hw), grid_project_bwd_row(), g_fc2_w, 2 * kProj,
                                    g_fc1_b, kProj, g_fc2_b, 2, acc_c, st),
             "reduce(fc2.weight | fc1.bias | fc2.bias)");
    int n_co = 0;
    FNO_CUDA((launch_grid_chan_outer<kProj, kC>(dz1, act + act_off, part_co, &n_co, nb, hw, st)), "grid_chan_outer_kernel(fc1)");
    FNO_CUDA(launch_reduce_partials(part_co, n_co, kProj * kC + kProj, g_fc1_w, kProj * kC, nullptr, 0, nullptr, 0, acc_c, st),
             "reduce(fc1.weight)");
  }
  return kOk;
}

int fno_grid_project_bwd(const float* act_in, const float* dpreds, const float* mask, const float* pre, const fno_weights* w,
                         float* dpre_out, float* dz1, float* partials, float* g_fc1_w, float* g_fc1_b, float* g_fc2_w,
                         float* g_fc2_b, int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_project_bwd", h, wd));
  if (!act_in || !dpreds || !mask || !pre || !w || !dpre_out || !dz1 || !partials || batch <= 0)
    return fail(kErrArg, "fno_grid_project_bwd: bad argument");
  const bool any = g_fc1_w || g_fc1_b || g_fc2_w || g_fc2_b, all = g_fc1_w && g_fc1_b && g_fc2_w && g_fc2_b;
  if (any && !all) return fail(kErrArg, "fno_grid_project_bwd: pass all four gradient pointers or none");
  FNO_ALIGN("fno_grid_project_bwd", act_in, 4);
  FNO_ALIGN("fno_grid_project_bwd", dpreds, 4);
  FNO_ALIGN("fno_grid_project_bwd", mask, 4);
  FNO_ALIGN("fno_grid_project_bwd", pre, 4);
  FNO_ALIGN("fno_grid_project_bwd", dpre_out, 4);
  FNO_ALIGN("fno_grid_project_bwd", dz1, 4);
  FNO_ALIGN("fno_grid_project_bwd", partials, 4);
  FNO_ALIGN("fno_grid_project_bwd", g_fc1_w, 4);
  FNO_ALIGN("fno_grid_project_bwd", g_fc1_b, 4);
  FNO_ALIGN("fno_grid_project_bwd", g_fc2_w, 4);
  FNO_ALIGN("fno_grid_project_bwd", g_fc2_b, 4);
  return grid_project_bwd_impl(act_in, dpreds, mask, pre, w, dpre_out, dz1, partials, g_fc1_w, g_fc1_b, g_fc2_w, g_fc2_b,
                               batch, h, wd, S(stream));
}

static int grid_block(const fno_weights* w, int l, const float* act_in, float* act_out, float* pre_out, void* xm,
                      const fno_workspace* ws, int batch, int h, int wd, void* stream) {
  const float inv = 1.f / static_cast<float>(h * wd);
  FNO_TRY(fno_grid_spectral_dft_fwd(act_in, xm, batch, h, wd, 1.f, 1.f, stream));
  FNO_TRY(fno_mode_mix(xm, w->spec_wk[l], ws->ym, batch, stream));
  FNO_TRY(fno_grid_spectral_inv_kx(ws->ym, static_cast<float*>(ws->z), batch, h, wd, inv, 2.f * inv, stream));
  return fno_grid_block_out(pre_out ? FNO_EPI_GELU_SAVE_PRE : FNO_EPI_GELU, static_cast<const float*>(ws->z), act_in,
                            w->w0t[l], w->w0_b[l], act_out, pre_out, nullptr, batch, h, wd, stream);
}

int fno_grid_forward(const fno_weights* w, const float* inputs, const float* mask, const float* case_params, float* preds,
                     const fno_workspace* ws, int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_forward", h, wd));
  if (!w || !ws || !ws->act[0] || !ws->act[1] || !ws->xm || !ws->ym || !ws->z) return fail(kErrArg, "fno_grid_forward: bad workspace");
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) return fail(kErrUnsupported, "fno_grid_forward: n_layers out of range");
  FNO_TRY(frames_align("fno_grid_forward", inputs, mask, case_params, 4));
  FNO_ALIGN("fno_grid_forward", preds, 4);
  float* act[2] = {static_cast<float*>(ws->act[0]), static_cast<float*>(ws->act[1])};
  FNO_TRY(fno_grid_lift_fwd(inputs, mask, case_params, w, act[0], batch, h, wd, stream));
  int cur = 0;
  for (int l = 0; l < w->n_layers; ++l) {
    FNO_TRY(grid_block(w, l, act[cur], act[cur ^ 1], nullptr, ws->xm, ws, batch, h, wd, stream));
    cur ^= 1;
  }
  return fno_grid_project_fwd(act[cur], mask, w, preds, batch, h, wd, stream);
}

static int grid_rollout_impl(const char* what, const fno_weights* w, const float* inputs, const float* mask,
                             const float* case_params, float* preds_seq, int steps, const fno_workspace* ws,
                             const fno_noise* nz, float* fed, int batch, int h, int wd, void* stream) {
  char msg[160];
  const fno_teacher* tc = nullptr;   // the inference rollout has no teacher
  FNO_TRY(grid_arg(what, h, wd));
  if (steps < 0 || !preds_seq || batch <= 0) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  FNO_TRY(frames_align(what, inputs, mask, case_params, 4));
  FNO_ALIGN(what, preds_seq, 4);
  FNO_ALIGN(what, fed, 4);
  const size_t frame = static_cast<size_t>(batch) * 2 * h * wd;
  const float* cur = inputs;
  for (int s = 0; s < steps; ++s) {
    float* nxt = preds_seq + static_cast<size_t>(s) * frame;
    FNO_TRY(feed_step(nz, tc, fed, mask, s, frame, batch, h, wd, cur, stream));
    FNO_TRY(fno_grid_forward(w, cur, mask, case_params, nxt, ws, batch, h, wd, stream));
    cur = nxt;
  }
  return kOk;
}

int fno_grid_rollout(const fno_weights* w, const float* inputs, const float* mask, const float* case_params, float* preds_seq,
                     int steps, const fno_workspace* ws, int batch, int h, int wd, void* stream) {
  return grid_rollout_impl("fno_grid_rollout", w, inputs, mask, case_params, preds_seq, steps, ws, nullptr, nullptr, batch, h,
                           wd, stream);
}

int fno_grid_rollout_noise(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                           float* preds_seq, int steps, const fno_workspace* ws, const fno_noise* noise, float* fed,
                           int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_rollout_noise", h, wd));
  FNO_TRY(noise_args("fno_grid_rollout_noise", noise, fed, steps));
  FNO_TRY(noise_forward_args("fno_grid_rollout_noise", w, inputs, mask, case_params, nullptr, ws, batch, true, 0));
  return grid_rollout_impl("fno_grid_rollout_noise", w, inputs, mask, case_params, preds_seq, steps, ws, noise, fed, batch, h,
                           wd, stream);
}

// fno_grid_forward_train up to the saved set (lift and Fourier blocks, no projection)
static int grid_forward_train_body(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                   const fno_train_saved* saved, const fno_workspace* ws, int batch, int h, int wd,
                                   void* stream) {
  FNO_TRY(fno_grid_lift_fwd(inputs, mask, case_params, w, static_cast<float*>(saved->act[0]), batch, h, wd, stream));
  for (int l = 0; l < w->n_layers; ++l) {
    if (!saved->act[l + 1] || !saved->pre[l] || !saved->xm[l])
      return fail(kErrArg, "fno_grid_forward_train: null saved buffer");
    FNO_TRY(grid_block(w, l, static_cast<const float*>(saved->act[l]), static_cast<float*>(saved->act[l + 1]), saved->pre[l],
                       saved->xm[l], ws, batch, h, wd, stream));
  }
  return kOk;
}

int fno_grid_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                           float* preds, const fno_train_saved* saved, const fno_workspace* ws, int batch, int h, int wd,
                           void* stream) {
  FNO_TRY(grid_arg("fno_grid_forward_train", h, wd));
  if (!w || !saved || !ws || !ws->ym || !ws->z || !saved->act[0]) return fail(kErrArg, "fno_grid_forward_train: bad argument");
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) return fail(kErrUnsupported, "fno_grid_forward_train: n_layers");
  FNO_TRY(frames_align("fno_grid_forward_train", inputs, mask, case_params, 4));
  FNO_ALIGN("fno_grid_forward_train", preds, 4);
  FNO_TRY(grid_forward_train_body(w, inputs, mask, case_params, saved, ws, batch, h, wd, stream));
  return fno_grid_project_fwd(static_cast<const float*>(saved->act[w->n_layers]), mask, w, preds, batch, h, wd, stream);
}

// The grid backward after argument checks; accum / hand_off / add / gate as in backward_impl (the rollout sweep's modes)
static int grid_backward_impl(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                              const float* case_params, const float* dpreds, const fno_train_saved* saved, const fno_grads* g,
                              const fno_bwd_scratch* sc, const fno_workspace* ws, float* d_inputs, float* d_case_params,
                              int batch, int h, int wd, void* stream, int accum = 0, int hand_off = 0,
                              const float* add = nullptr, const unsigned char* gate = nullptr) {
  cudaStream_t st = S(stream);
  const int L = w->n_layers, p = w->n_case_params;
  // ---- projection -> d[0] = dpre_{L-1}
  FNO_TRY(grid_project_bwd_impl(static_cast<const float*>(saved->act[L]), dpreds, mask, saved->pre[L - 1], w, sc->d[0], sc->dz1,
                                sc->partials, g ? g->fc1_w : nullptr, g ? g->fc1_b : nullptr, g ? g->fc2_w : nullptr,
                                g ? g->fc2_b : nullptr, batch, h, wd, st, accum));
  // ---- Fourier blocks, last to first
  float* part_co = sc->partials + grid_partials_offset_co();
  const float inv = 1.f / static_cast<float>(h * wd);
  int cur = 0;
  for (int l = L - 1; l >= 0; --l) {
    float* dpre = sc->d[cur];
    float* dnext = sc->d[cur ^ 1];
    const float* act_l = static_cast<const float*>(saved->act[l]);
    if (g) {
      int n_co = 0;
      FNO_CUDA((launch_grid_chan_outer<kC, kC>(dpre, act_l, part_co, &n_co, batch, h * wd, st)), "grid_chan_outer_kernel(w0)");
      FNO_CUDA(launch_reduce_partials(part_co, n_co, kC * kC + kC, g->w0_w[l], kC * kC, g->w0_b[l], kC, nullptr, 0, accum, st),
               "reduce(w0.weight | w0.bias)");
    }
    FNO_TRY(fno_grid_spectral_dft_fwd(dpre, sc->gm, batch, h, wd, inv, 2.f * inv, stream));
    if (g) {
      FNO_CUDA(launch_spectral_wgrad(saved->xm[l], sc->gm, sc->gwk, batch, st), "spectral_wgrad_kernel");
      FNO_CUDA(launch_unpack_spectral(sc->gwk, g->spec_w1[l], g->spec_w2[l], accum, st), "unpack_spectral_kernel");
    }
    FNO_TRY(fno_mode_mix(sc->gm, wb->spec_wkT[l], ws->ym, batch, stream));
    FNO_TRY(fno_grid_spectral_inv_kx(ws->ym, static_cast<float*>(ws->z), batch, h, wd, 1.f, 1.f, stream));
    FNO_TRY(fno_grid_block_out(l > 0 ? FNO_EPI_MUL_DGELU : FNO_EPI_PLAIN, static_cast<const float*>(ws->z), dpre, wb->w0[l],
                               nullptr, dnext, nullptr, l > 0 ? saved->pre[l - 1] : nullptr, batch, h, wd, stream));
    cur ^= 1;
  }
  // ---- lift: fc0 gradients and the data adjoint of dL/da0 = d[cur]
  float* part_lb = g ? sc->partials + grid_partials_offset_lb() : nullptr;
  if (g || d_inputs || d_case_params) {
    FNO_CUDA(launch_grid_lift_bwd(sc->d[cur], inputs, mask, case_params, w->gx, w->gy, w->fc0_w, part_lb, d_inputs,
                                  d_case_params, hand_off ? add : nullptr, hand_off, batch, p, h, wd, st,
                                  hand_off ? gate : nullptr),
             "grid_lift_bwd_kernel");
  }
  if (g)
    FNO_CUDA(launch_reduce_partials(part_lb, grid_lift_bwd_parts(batch), grid_lift_bwd_row(), g->fc0_w, kC * (5 + p), g->fc0_b,
                                    kC, nullptr, 0, accum, st),
             "reduce(fc0.weight | fc0.bias)");
  return kOk;
}

int fno_grid_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                      const float* case_params, const float* dpreds, const fno_train_saved* saved, const fno_grads* g,
                      const fno_bwd_scratch* sc, const fno_workspace* ws, float* d_inputs, float* d_case_params, int batch,
                      int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_backward", h, wd));
  if (!w || !wb || !inputs || !mask || !dpreds || !saved || !sc || !ws || batch <= 0)
    return fail(kErrArg, "fno_grid_backward: bad argument");
  if (w->n_layers < 1 || w->n_layers > FNO_MAX_LAYERS) return fail(kErrUnsupported, "fno_grid_backward: n_layers");
  if (w->n_case_params < 0 || w->n_case_params > kMaxCaseParams)
    return fail(kErrArg, "fno_grid_backward: n_case_params out of range");
  if (w->n_case_params == 0) d_case_params = nullptr;   // nothing to write
  if (!g && !d_inputs && !d_case_params) return fail(kErrArg, "fno_grid_backward: no output requested");
  if (!sc->d[0] || !sc->d[1] || !sc->dz1 || !sc->gm || !sc->gwk || !sc->partials || !ws->ym || !ws->z)
    return fail(kErrArg, "fno_grid_backward: null scratch buffer");
  FNO_TRY(frames_align("fno_grid_backward", inputs, mask, case_params, 4));
  FNO_ALIGN("fno_grid_backward", dpreds, 4);
  FNO_ALIGN("fno_grid_backward", d_inputs, 4);
  FNO_ALIGN("fno_grid_backward", d_case_params, 4);
  return grid_backward_impl(w, wb, inputs, mask, case_params, dpreds, saved, g, sc, ws, d_inputs, d_case_params, batch, h, wd,
                            stream);
}

static int grid_rollout_forward_train_impl(const char* what, const fno_weights* w, const float* inputs, const float* mask,
                                           const float* case_params, float* preds_seq, int steps,
                                           const fno_train_saved* saved, const fno_workspace* ws, const fno_noise* nz,
                                           const fno_teacher* tc, float* fed, int batch, int h, int wd, void* stream) {
  char msg[160];
  FNO_TRY(grid_arg(what, h, wd));
  if (steps < 1 || !inputs || !preds_seq || batch <= 0) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  FNO_TRY(frames_align(what, inputs, mask, case_params, 4));
  FNO_ALIGN(what, preds_seq, 4);
  FNO_ALIGN(what, fed, 4);
  const size_t frame = static_cast<size_t>(batch) * 2 * h * wd;
  const float* cur = inputs;
  for (int s = 0; s < steps; ++s) {
    float* nxt = preds_seq + static_cast<size_t>(s) * frame;
    FNO_TRY(feed_step(nz, tc, fed, mask, s, frame, batch, h, wd, cur, stream));
    FNO_TRY(fno_grid_forward_train(w, cur, mask, case_params, nxt, saved, ws, batch, h, wd, stream));
    cur = nxt;
  }
  return kOk;
}

int fno_grid_rollout_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                   float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws,
                                   int batch, int h, int wd, void* stream) {
  return grid_rollout_forward_train_impl("fno_grid_rollout_forward_train", w, inputs, mask, case_params, preds_seq, steps,
                                         saved, ws, nullptr, nullptr, nullptr, batch, h, wd, stream);
}

int fno_grid_rollout_forward_train_noise(const fno_weights* w, const float* inputs, const float* mask,
                                         const float* case_params, float* preds_seq, int steps, const fno_train_saved* saved,
                                         const fno_workspace* ws, const fno_noise* noise, float* fed, int batch, int h, int wd,
                                         void* stream) {
  FNO_TRY(grid_arg("fno_grid_rollout_forward_train_noise", h, wd));
  FNO_TRY(noise_args("fno_grid_rollout_forward_train_noise", noise, fed, steps));
  FNO_TRY(noise_forward_args("fno_grid_rollout_forward_train_noise", w, inputs, mask, case_params, saved, ws, batch, true,
                             0));
  return grid_rollout_forward_train_impl("fno_grid_rollout_forward_train_noise", w, inputs, mask, case_params, preds_seq,
                                         steps, saved, ws, noise, nullptr, fed, batch, h, wd, stream);
}

int fno_grid_rollout_forward_train_feed(const fno_weights* w, const float* inputs, const float* mask,
                                        const float* case_params, float* preds_seq, int steps, const fno_train_saved* saved,
                                        const fno_workspace* ws, const fno_noise* noise, const fno_teacher* teacher, float* fed,
                                        int batch, int h, int wd, void* stream) {
  const char* what = "fno_grid_rollout_forward_train_feed";
  FNO_TRY(grid_arg(what, h, wd));
  if (noise) FNO_TRY(noise_args(what, noise, fed, steps));
  FNO_TRY(teacher_args(what, teacher, fed, true));
  FNO_TRY(noise_forward_args(what, w, inputs, mask, case_params, saved, ws, batch, true, 0));
  return grid_rollout_forward_train_impl(what, w, inputs, mask, case_params, preds_seq, steps, saved, ws, noise, teacher, fed,
                                         batch, h, wd, stream);
}

static int grid_rollout_backward_impl(const char* what, const fno_weights* w, const fno_weights_bwd* wb, const float* inputs,
                                      const float* mask, const float* case_params, const float* preds_seq,
                                      const float* dpreds_seq, int steps, const fno_train_saved* saved, const fno_grads* grads,
                                      const fno_bwd_scratch* scratch, const fno_workspace* ws, const fno_noise* nz,
                                      const fno_teacher* tc, const float* fed, float* carry, float* d_inputs,
                                      float* d_case_params, int batch, int h, int wd, void* stream) {
  char msg[160];
  FNO_TRY(grid_arg(what, h, wd));
  if (w && w->n_case_params == 0) d_case_params = nullptr;   // nothing to write
  FNO_TRY(rollout_bwd_args(what, w, wb, inputs, mask, preds_seq, dpreds_seq, steps, saved, grads, scratch, ws, carry, d_inputs,
                           d_case_params, batch));
  if (!saved->act[0]) {
    snprintf(msg, sizeof(msg), "%s: null saved buffer", what);
    return fail(kErrArg, msg);
  }
  FNO_TRY(frames_align(what, inputs, mask, case_params, 4));
  FNO_ALIGN(what, preds_seq, 4);
  FNO_ALIGN(what, dpreds_seq, 4);
  FNO_ALIGN(what, fed, 4);
  FNO_ALIGN(what, carry, 4);
  FNO_ALIGN(what, d_inputs, 4);
  FNO_ALIGN(what, d_case_params, 4);
  const size_t frame = static_cast<size_t>(batch) * 2 * h * wd;
  if (d_case_params)   // every sweep step adds its share
    FNO_CUDA(cudaMemsetAsync(d_case_params, 0, static_cast<size_t>(batch) * w->n_case_params * sizeof(float), S(stream)),
             "memset(d_case_params)");
  for (int s = steps - 1; s >= 0; --s) {
    const float* x = fed_frame(nz, tc, fed, inputs, preds_seq, s, frame);
    FNO_TRY(grid_forward_train_body(w, x, mask, case_params, saved, ws, batch, h, wd, stream));
    const float* up = s == steps - 1 ? dpreds_seq + static_cast<size_t>(s) * frame : carry;
    FNO_TRY(grid_backward_impl(w, wb, x, mask, case_params, up, saved, grads, scratch, ws, s > 0 ? carry : d_inputs,
                               d_case_params, batch, h, wd, stream, s != steps - 1 ? 1 : 0, 1,
                               s > 0 ? dpreds_seq + static_cast<size_t>(s - 1) * frame : nullptr,
                               tc && s > 0 ? tc->flags + static_cast<size_t>(s - 1) * batch : nullptr));
  }
  return kOk;
}

int fno_grid_rollout_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                              const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                              const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                              const fno_workspace* ws, float* carry, float* d_inputs, float* d_case_params, int batch, int h,
                              int wd, void* stream) {
  return grid_rollout_backward_impl("fno_grid_rollout_backward", w, wb, inputs, mask, case_params, preds_seq, dpreds_seq, steps,
                                    saved, grads, scratch, ws, nullptr, nullptr, nullptr, carry, d_inputs, d_case_params, batch,
                                    h, wd, stream);
}

int fno_grid_rollout_backward_noise(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                                    const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                                    const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                                    const fno_workspace* ws, const fno_noise* noise, const float* fed, float* carry,
                                    float* d_inputs, float* d_case_params, int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_rollout_backward_noise", h, wd));
  FNO_TRY(noise_args("fno_grid_rollout_backward_noise", noise, fed, steps));
  return grid_rollout_backward_impl("fno_grid_rollout_backward_noise", w, wb, inputs, mask, case_params, preds_seq, dpreds_seq,
                                    steps, saved, grads, scratch, ws, noise, nullptr, fed, carry, d_inputs, d_case_params,
                                    batch, h, wd, stream);
}

int fno_grid_rollout_backward_feed(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                                   const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                                   const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                                   const fno_workspace* ws, const fno_noise* noise, const fno_teacher* teacher,
                                   const float* fed, float* carry, float* d_inputs, float* d_case_params, int batch, int h,
                                   int wd, void* stream) {
  const char* what = "fno_grid_rollout_backward_feed";
  FNO_TRY(grid_arg(what, h, wd));
  if (noise) FNO_TRY(noise_args(what, noise, fed, steps));
  FNO_TRY(teacher_args(what, teacher, fed, false));
  return grid_rollout_backward_impl(what, w, wb, inputs, mask, case_params, preds_seq, dpreds_seq, steps, saved, grads, scratch,
                                    ws, noise, teacher, fed, carry, d_inputs, d_case_params, batch, h, wd, stream);
}

int fno_grid_multistep_metrics(const float* preds_seq, const float* label_u, const float* mask, float* sums, int steps,
                               int batch, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_multistep_metrics", h, wd));
  if (!preds_seq || !label_u || !mask || !sums || steps <= 0 || steps > 65535 || batch <= 0)
    return fail(kErrArg, "fno_grid_multistep_metrics: bad argument");
  FNO_ALIGN("fno_grid_multistep_metrics", preds_seq, 4);
  FNO_ALIGN("fno_grid_multistep_metrics", label_u, 4);
  FNO_ALIGN("fno_grid_multistep_metrics", mask, 4);
  FNO_ALIGN("fno_grid_multistep_metrics", sums, 4);
  FNO_CUDA(launch_grid_multistep_metrics(preds_seq, label_u, mask, sums, steps, batch, h, wd, S(stream)),
           "grid_multistep_metrics_kernel");
  return kOk;
}

int fno_grid_gather_batch(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                          const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                          float* mask, float* case_params, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_gather_batch", h, wd));
  if (!frames_in || !frames_out || !case_ids || !idx || !inputs || !label || !mask || n_idx <= 0 || n_case_params < 0 ||
      n_case_params > kMaxCaseParams || bad_dtype(frame_dtype) || (n_case_params > 0 && (!case_table || !case_params)))
    return fail(kErrArg, "fno_grid_gather_batch: bad argument");
  FNO_TRY(gather_align("fno_grid_gather_batch", frames_in, frames_out, case_table, case_ids, idx, frame_dtype, inputs, label,
                       mask, case_params, nullptr, false));
  FNO_CUDA(launch_grid_gather_batch(frames_in, frames_out, case_table, reinterpret_cast<const int*>(case_ids),
                                    reinterpret_cast<const long long*>(idx), n_idx, n_case_params,
                                    frame_dtype == FNO_ACT_BF16, inputs, label, mask, case_params, h, wd, S(stream)),
           "grid_gather_batch_kernel");
  return kOk;
}

int fno_grid_gather_window(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                           const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                           float* mask, float* case_params, int steps, int time_step_size, int64_t n_frames,
                           float* labels_seq, int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_gather_window", h, wd));
  FNO_TRY(gather_window_args("fno_grid_gather_window", frames_in, frames_out, case_table, case_ids, idx, n_idx,
                             n_case_params, frame_dtype, inputs, mask, case_params, steps, time_step_size, n_frames,
                             labels_seq));
  FNO_TRY(gather_align("fno_grid_gather_window", frames_in, frames_out, case_table, case_ids, idx, frame_dtype, inputs, label,
                       mask, case_params, labels_seq, false));
  FNO_CUDA(launch_grid_gather_window(frames_in, frames_out, case_table, reinterpret_cast<const int*>(case_ids),
                                     reinterpret_cast<const long long*>(idx), n_idx, n_case_params,
                                     frame_dtype == FNO_ACT_BF16, inputs, label, mask, case_params, steps, time_step_size,
                                     n_frames, labels_seq, h, wd, S(stream)),
           "gather_window_kernel");
  return kOk;
}

int fno_add_input_noise(float* inputs, const float* mask, const int64_t* idx, int n, int h, int wd, float std,
                        uint64_t seed, const int64_t* step_base, const int32_t* step_offset, void* stream) {
  FNO_TRY(grid_arg("fno_add_input_noise", h, wd));
  if (!inputs || !mask || !idx || !step_base || n <= 0 || !(std >= 0.f) || !isfinite(std))
    return fail(kErrArg, "fno_add_input_noise: bad argument");
  FNO_ALIGN("fno_add_input_noise", inputs, 4);   // float4 only where both frames are 16-byte aligned
  FNO_ALIGN("fno_add_input_noise", mask, 4);
  FNO_ALIGN("fno_add_input_noise", idx, 8);
  FNO_ALIGN("fno_add_input_noise", step_base, 8);
  FNO_ALIGN("fno_add_input_noise", step_offset, 4);
  FNO_CUDA(launch_add_input_noise(inputs, mask, reinterpret_cast<const long long*>(idx), n, h, wd, std, seed,
                                  reinterpret_cast<const long long*>(step_base), reinterpret_cast<const int*>(step_offset),
                                  S(stream)),
           "add_input_noise_kernel");
  return kOk;
}

int fno_add_input_noise_stream(const float* in, float* out, const float* mask, const int64_t* idx, int n, int h, int wd,
                               float std, uint64_t seed, const int64_t* step_base, const int32_t* step_offset,
                               int noise_stream, void* stream) {
  FNO_TRY(grid_arg("fno_add_input_noise_stream", h, wd));
  if (!in || !out || !mask || !idx || !step_base || n <= 0 || !(std >= 0.f) || !isfinite(std) || noise_stream < 0 ||
      noise_stream >= FNO_NOISE_STREAMS)
    return fail(kErrArg, "fno_add_input_noise_stream: bad argument");
  FNO_ALIGN("fno_add_input_noise_stream", in, 4);   // float4 only where the frames are 16-byte aligned
  FNO_ALIGN("fno_add_input_noise_stream", out, 4);
  FNO_ALIGN("fno_add_input_noise_stream", mask, 4);
  FNO_ALIGN("fno_add_input_noise_stream", idx, 8);
  FNO_ALIGN("fno_add_input_noise_stream", step_base, 8);
  FNO_ALIGN("fno_add_input_noise_stream", step_offset, 4);
  FNO_CUDA(launch_input_noise_stream(in, out, mask, reinterpret_cast<const long long*>(idx), n, h, wd, std, seed,
                                     reinterpret_cast<const long long*>(step_base), reinterpret_cast<const int*>(step_offset),
                                     noise_stream, S(stream)),
           "input_noise_stream_kernel");
  return kOk;
}

int fno_teacher_flags(const int64_t* idx, int batch, int steps, const float* prob, uint64_t seed, const int64_t* step_base,
                      const int32_t* step_offset, uint8_t* flags, void* stream) {
  if (!idx || !prob || !step_base || !flags || batch <= 0 || steps < 2 || steps > FNO_NOISE_STREAMS ||
      static_cast<long long>(steps - 1) * batch > 0x7fffffffll)
    return fail(kErrArg, "fno_teacher_flags: bad argument");
  FNO_ALIGN("fno_teacher_flags", idx, 8);
  FNO_ALIGN("fno_teacher_flags", prob, 4);
  FNO_ALIGN("fno_teacher_flags", step_base, 8);
  FNO_ALIGN("fno_teacher_flags", step_offset, 4);
  FNO_CUDA(launch_teacher_flags(reinterpret_cast<const long long*>(idx), batch, steps, prob, seed,
                                reinterpret_cast<const long long*>(step_base), reinterpret_cast<const int*>(step_offset),
                                flags, S(stream)),
           "teacher_flags_kernel");
  return kOk;
}

int fno_eval_sums(const float* preds, const float* label, const float* mask, const float* inputs, float* sums, int batch,
                  int h, int wd, void* stream) {
  FNO_TRY(grid_arg("fno_eval_sums", h, wd));
  if (!preds || !label || !mask || !inputs || !sums || batch <= 0) return fail(kErrArg, "fno_eval_sums: bad argument");
  FNO_ALIGN("fno_eval_sums", preds, 4);
  FNO_ALIGN("fno_eval_sums", label, 4);
  FNO_ALIGN("fno_eval_sums", mask, 4);
  FNO_ALIGN("fno_eval_sums", inputs, 4);
  FNO_ALIGN("fno_eval_sums", sums, 4);
  FNO_CUDA(launch_eval_sums(preds, label, mask, inputs, sums, batch, h, wd, S(stream)), "eval_sums_kernel");
  return kOk;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ window rollout metrics
static int window_metrics_args(const char* what, const float* preds_seq, const void* frames_in, const void* frames_out,
                               const int64_t* starts, int steps, int batch, int time_step_size, int64_t n_frames,
                               int frame_dtype, const float* sums) {
  char msg[160];
  if (!preds_seq || !frames_in || !frames_out || !starts || !sums || steps < 1 || steps > 65535 || batch < 1 ||
      time_step_size < 1 || n_frames < 1 || bad_dtype(frame_dtype)) {
    snprintf(msg, sizeof(msg), "%s: bad argument", what);
    return fail(kErrArg, msg);
  }
  return kOk;
}

int fno_window_metrics(const float* preds_seq, const void* frames_in, const void* frames_out, const int64_t* starts,
                       int steps, int batch, int time_step_size, int64_t n_frames, int frame_dtype, float* sums,
                       void* stream) {
  FNO_TRY(window_metrics_args("fno_window_metrics", preds_seq, frames_in, frames_out, starts, steps, batch, time_step_size,
                              n_frames, frame_dtype, sums));
  // the 64x64 kernel's vector loads: float4 predictions, four frame elements at a time
  FNO_ALIGN("fno_window_metrics", preds_seq, 16);
  FNO_ALIGN("fno_window_metrics", frames_in, frame_vec_bytes(frame_dtype));
  FNO_ALIGN("fno_window_metrics", frames_out, frame_vec_bytes(frame_dtype));
  FNO_ALIGN("fno_window_metrics", starts, 8);
  FNO_ALIGN("fno_window_metrics", sums, 4);
  FNO_CUDA(launch_window_metrics(preds_seq, frames_in, frames_out, reinterpret_cast<const long long*>(starts), steps, batch,
                                 time_step_size, n_frames, frame_dtype == FNO_ACT_BF16, sums, S(stream)),
           "window_metrics_kernel");
  return kOk;
}

int fno_grid_window_metrics(const float* preds_seq, const void* frames_in, const void* frames_out, const int64_t* starts,
                            int steps, int batch, int time_step_size, int64_t n_frames, int frame_dtype, float* sums, int h,
                            int wd, void* stream) {
  FNO_TRY(grid_arg("fno_grid_window_metrics", h, wd));
  FNO_TRY(window_metrics_args("fno_grid_window_metrics", preds_seq, frames_in, frames_out, starts, steps, batch,
                              time_step_size, n_frames, frame_dtype, sums));
  FNO_ALIGN("fno_grid_window_metrics", preds_seq, 4);
  FNO_ALIGN("fno_grid_window_metrics", frames_in, frame_dtype == FNO_ACT_BF16 ? 2u : 4u);
  FNO_ALIGN("fno_grid_window_metrics", frames_out, frame_dtype == FNO_ACT_BF16 ? 2u : 4u);
  FNO_ALIGN("fno_grid_window_metrics", starts, 8);
  FNO_ALIGN("fno_grid_window_metrics", sums, 4);
  FNO_CUDA(launch_grid_window_metrics(preds_seq, frames_in, frames_out, reinterpret_cast<const long long*>(starts), steps,
                                      batch, time_step_size, n_frames, frame_dtype == FNO_ACT_BF16, sums, h, wd, S(stream)),
           "window_metrics_kernel");
  return kOk;
}
