/* cfdbench_b200 -- C ABI of the H100-native FNO hot path for CFDBench.
 *
 * The reference (luo-yining/CFDBench @ 6c30c62) is pure Python/PyTorch: its "FFI" for this path is the
 * set of ATen calls made by src/models/fno/fno2d.py.  Each entry point below replaces the calls cited
 * next to it.  All pointers are raw device pointers unless a name ends in _host; buffers are owned by the
 * caller (PyTorch's allocator in the Python wrapper); every call is asynchronous on `stream`
 * (a cudaStream_t passed as void*) and returns 0 on success, non-zero otherwise
 * (fno_last_error() gives the message).  No entry point synchronises the device, none falls back to CPU.
 *
 * Fixed configuration (the reference's FNO config, src/args.py:99-103,187-197): H=W=64, hidden=32,
 * modes 12x12, fc1 width 128, out_chan=2, in_chan=2.  Other grids (24 <= H, W <= 128, e.g. the 66x65 tube and dam
 * frames) go through the fno_grid_* entry points at the end of this header (fp32 storage only).  Activation storage `act_dtype`:
 * FNO_ACT_F32 (parity mode) or FNO_ACT_BF16 (hidden activations stored as bf16 between kernels);
 * arithmetic is fp32 in both.
 *
 * Layouts
 *   activations      [B][32][64][64]   act_dtype, NCHW contiguous
 *   frames / preds   [B][2][64][64]    float32
 *   mask             [B][64][64]       float32  (a (B,1,64,64) tensor has the same layout)
 *   case_params      [B][p]            float32
 *   modes (xm, ym)   [288][B][32]      complex64 (interleaved re,im), MODE-major; mode k = kxi*12 + ky,
 *                                      kxi 0..11 <-> kx 0..11 (weights1), kxi 12..23 <-> kx 52..63 (weights2)
 *   packed spectral  [288][32 in][32 out] complex64 (fno_pack_spectral_weights)
 *   mix operand      per mode 2 x [64 = (out, re|im)][64 = (in, re|im)] float32: the real-expanded block as tf32
 *                    hi / lo images in the tensor core's K-major operand layout (fno_pack_mix_operand)
 *   w0t              [32 in][32 out]   float32  (transpose of the Conv2d weight (out,in,1,1))
 */
#ifndef CFDBENCH_B200_H_
#define CFDBENCH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FNO_ABI_VERSION 4
#define FNO_MAX_LAYERS 8

enum { FNO_ACT_F32 = 0, FNO_ACT_BF16 = 1 };
/* epilogues of fno_block_out */
enum { FNO_EPI_GELU = 0, FNO_EPI_GELU_SAVE_PRE = 1, FNO_EPI_MUL_DGELU = 2, FNO_EPI_PLAIN = 3 };

/* Device-side weights of one model, in kernel layouts (built by the fno_pack_* calls). */
typedef struct fno_weights {
  int32_t n_layers;      /* reference fno_depth (4) */
  int32_t n_case_params; /* p: 5 cavity, 8 cylinder (reference src/utils/autoregressive.py:31-37) */
  const float* fc0_w;    /* [32][5+p]  fc0.weight  (reference fno2d.py:150-156) */
  const float* fc0_b;    /* [32] */
  const void* spec_wk[FNO_MAX_LAYERS]; /* mix operand of blocks.{l}.conv0.weights1/2 (fno_pack_mix_operand) */
  const float* w0t[FNO_MAX_LAYERS];    /* blocks.{l}.w0.weight transposed */
  const float* w0_b[FNO_MAX_LAYERS];   /* blocks.{l}.w0.bias */
  const float* fc1_w;    /* [128][32] fc1.weight */
  const float* fc1_b;    /* [128] */
  const float* fc2_w;    /* [2][128]  fc2.weight */
  const float* fc2_b;    /* [2] */
  const float* gx;       /* [64] float32(np.linspace(0,1,64)): x coordinate per row h (fno2d.py:244-255) */
  const float* gy;       /* [64] y coordinate per column w */
} fno_weights;

/* Caller-provided scratch for a batch of B samples. */
typedef struct fno_workspace {
  void* act[2]; /* two activation buffers, B*32*4096 elements of act_dtype each (ping-pong) */
  void* xm;     /* B*288*32 complex64 */
  void* ym;     /* B*288*32 complex64 */
  void* z;      /* B*64*24*32 float32: rows of the half-inverted spectrum, Z[b][h][2 ky + (re|im)][o] */
  void* ym_img; /* fno_ym_image_bytes(B), or NULL.  When set and act_dtype == FNO_ACT_BF16, inference blocks take the
                 * fused output stage (fno_mode_mix_image + fno_block_fused) and `ym` / `z` are not touched. */
} fno_workspace;

int fno_version(void);
/* Frees what the library itself owns on the CURRENT device (constant operand tables built on first use); they are
 * rebuilt on demand.  Everything else is caller-owned.  Synchronises the device. */
int fno_destroy(void);
const char* fno_last_error(void);
/* bytes of one activation buffer / one mode buffer for batch B */
size_t fno_act_bytes(int batch, int act_dtype);
size_t fno_modes_bytes(int batch);
size_t fno_z_bytes(int batch);
size_t fno_ym_image_bytes(int batch);
size_t fno_bwd_partials_bytes(void);

/* weights1, weights2: (32,32,12,12) complex64 as stored by the reference (fno2d.py:31-51).
 * conj_transpose=0 -> wk[k][i][o] = W[i][o][k] (forward); 1 -> wk[k][o][i] = conj(W[i][o][k]) (adjoint). */
int fno_pack_spectral_weights(const void* weights1, const void* weights2, void* wk, int conj_transpose, void* stream);
/* packed weights wk[288][32][32] -> the operand image fno_mode_mix consumes (fno_mix_operand_bytes() bytes).
 * Run once per weight update; for the adjoint mix feed it the conj_transpose=1 pack. */
size_t fno_mix_operand_bytes(void);
int fno_pack_mix_operand(const void* wk, void* wop, void* stream);
/* both steps in one launch: weights1/weights2 -> operand image (what the module runs after every optimizer step) */
int fno_pack_mix_operand_from_weights(const void* weights1, const void* weights2, void* wop, int conj_transpose,
                                      void* stream);
/* gradient wrt packed forward weights [288][32][32] -> gradients of weights1 / weights2 */
int fno_unpack_spectral_grads(const void* gwk, void* gw1, void* gw2, void* stream);

/* Channel assembly + fc0: torch.cat/repeat/get_coords/Conv2d(5+p,32,1) (reference fno2d.py:195-217,244-255) */
int fno_lift_fwd(const float* inputs, const float* mask, const float* case_params, const fno_weights* w,
                 void* act_out, int batch, int act_dtype, void* stream);

/* The four phases of SpectralConv2d_fast + FnoBlock (reference fno2d.py:59-82, 106-112):            */
/* (1) torch.fft.rfft2 restricted to the kept modes (fno2d.py:62,73-78); outputs scaled by s0 (ky=0), s1 (ky>0).
 *     fp32 planes: register FFT codelets (fno_dft_fwd.cu); bf16 planes: two chained tensor-core GEMMs
 *     (fno_dft_fwd_tc.cu: 37 us per launch at B=256 on an H100 80GB HBM3 (SXM) at a 700 W power limit, launched
 *     back to back; same 2e-6 against float64). */
int fno_spectral_dft_fwd(const void* act_in, void* xm, int batch, int act_dtype, float s0, float s1, void* stream);
/* (2) einsum("bixy,ioxy->boxy") on both corners (fno2d.py:54-57,73-78); wop = fno_pack_mix_operand image */
int fno_mode_mix(const void* xm, const void* wop, void* ym, int batch, void* stream);
/* (3) first half of irfft2 on the zero-padded spectrum (fno2d.py:65-72,81): inverse C2C along kx of the 24 kept
 *     rows, scaled by s0 (ky=0) / s1 (ky>0) (forward: 1/4096, 2/4096): z[b][h][2 ky + (re|im)][o], fno_z_bytes(B). */
int fno_spectral_inv_kx(const void* ym, void* z, int batch, float s0, float s1, void* stream);
/* (4) second half of irfft2 (C2R along ky, Im of the ky=0 column dropped) + Conv2d(32,32,1) + add + GELU
 *     (fno2d.py:81,104-111) as one tensor-core GEMM per 128-pixel tile.  pre_out/pre_in: see FNO_EPI_*. */
int fno_block_out(int epilogue, const void* z, const void* act_in, const float* w0t, const float* bias, void* act_out,
                  float* pre_out, const float* pre_in, int batch, int act_dtype, void* stream);
/* bf16 storage, inference: the output stage of a Fourier block in ONE kernel (block_fused_kernel, fno_block_fused.cu)
 * -- replaces fno_spectral_inv_kx + fno_block_out(FNO_EPI_GELU), i.e. irfft2 + Conv2d(32,32,1) + add + GELU of
 * reference src/models/fno/fno2d.py:81,104-111, without the Z round trip through HBM.
 *   fno_mode_mix_image: same product as fno_mode_mix, written as the per-sample tensor-core operand image the fused
 *     kernel bulk-copies (tf32 hi/lo split, fno_ym_image_bytes(B) bytes).
 *   fno_block_fused:    act_out = GELU(irfft2(pad(Y)) + W0 act_in + bias); act_in / act_out bf16 [B][32][64][64],
 *     16-byte aligned (they are read and written by TMA). */
int fno_mode_mix_image(const void* xm, const void* wop, void* ym_img, int batch, void* stream);
int fno_block_fused(const void* ym_img, const void* act_in_bf16, const float* w0t, const float* bias, void* act_out_bf16,
                    int batch, void* stream);
/* all four: act_out = FnoBlock_l(act_in) */
int fno_block_fwd(const fno_weights* w, int layer, const void* act_in, void* act_out, float* pre_out,
                  const fno_workspace* ws, int batch, int act_dtype, void* stream);

/* fc1 + GELU + fc2 + "* mask" (reference fno2d.py:228-233) */
int fno_project_fwd(const void* act_in, const float* mask, const fno_weights* w, float* preds, int batch,
                    int act_dtype, void* stream);

/* Fno2d.forward without the loss (reference fno2d.py:178-233): preds[B][2][64][64] */
int fno_forward(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                float* preds, const fno_workspace* ws, int batch, int act_dtype, void* stream);

/* Fno2d.generate_many (reference fno2d.py:269-295): preds_seq[steps][B][2][64][64], step s feeds step s+1 */
int fno_rollout(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                float* preds_seq, int steps, const fno_workspace* ws, int batch, int act_dtype, void* stream);

/* Same, with HOST buffers (pinned or pageable): copies inputs/mask/case_params to the device scratch
 * frames `dev_io` (caller-provided: (2 + 1 + steps*2)*B*4096*4 + B*p*4 bytes), runs the rollout and copies
 * preds_seq back; returns after the D2H copy has been enqueued (synchronise the stream to read). */
int fno_rollout_host(const fno_weights* w, const float* inputs_host, const float* mask_host,
                     const float* case_params_host, float* preds_seq_host, int steps, const fno_workspace* ws,
                     void* dev_io, int batch, int act_dtype, void* stream);
size_t fno_rollout_host_scratch_bytes(int batch, int n_case_params, int steps);

/* ---------------------------------------------------------------------------------------------------
 * Training step (what torch.autograd derives for loss["nmse"].backward(), reference src/train_auto.py:255)
 * ------------------------------------------------------------------------------------------------- */

/* Buffers the forward pass leaves for the backward pass (caller-allocated, batch B). */
typedef struct fno_train_saved {
  void* act[FNO_MAX_LAYERS + 1]; /* a_0 (lift output) .. a_L (last block output), act_dtype */
  float* pre[FNO_MAX_LAYERS];    /* pre-activation of each block, float32 [B][32][64][64] */
  void* xm[FNO_MAX_LAYERS];      /* kept modes of a_l, complex64 [288][B][32] */
} fno_train_saved;

/* Extra weight views the backward pass needs. */
typedef struct fno_weights_bwd {
  const void* spec_wkT[FNO_MAX_LAYERS]; /* mix operand of fno_pack_spectral_weights(..., conj_transpose=1) */
  const float* w0[FNO_MAX_LAYERS];      /* blocks.{l}.w0.weight in its natural [out][in] layout */
} fno_weights_bwd;

/* Gradient outputs, reference parameter layouts (float32 / complex64). All are overwritten. */
typedef struct fno_grads {
  float* fc0_w; /* [32][5+p] */
  float* fc0_b; /* [32] */
  void* spec_w1[FNO_MAX_LAYERS]; /* (32,32,12,12) complex64 */
  void* spec_w2[FNO_MAX_LAYERS];
  float* w0_w[FNO_MAX_LAYERS]; /* [32][32] */
  float* w0_b[FNO_MAX_LAYERS]; /* [32] */
  float* fc1_w; /* [128][32] */
  float* fc1_b; /* [128] */
  float* fc2_w; /* [2][128] */
  float* fc2_b; /* [2] */
} fno_grads;

/* Scratch of the backward pass. */
typedef struct fno_bwd_scratch {
  float* d[2];   /* two float32 [B][32][64][64] gradient buffers (ping-pong) */
  float* dz1;    /* float32 [min(B,FNO_BWD_CHUNK)][128][64][64] */
  void* gm;      /* complex64 [288][B][32] (mode-major): scaled modes of the block's upstream gradient */
  void* gwk;     /* complex64 [288][32][32] */
  float* partials; /* fno_bwd_partials_bytes() bytes: per-CTA shares of the small gradients (fc0/fc1/fc2/w0), summed in a
                    * fixed order by a second launch instead of float atomics -> bit-reproducible gradients */
} fno_bwd_scratch;
#define FNO_BWD_CHUNK 32

/* Fno2d.forward (reference fno2d.py:178-233) that also fills `saved`. ws->ym is used as scratch. */
int fno_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                      float* preds, const fno_train_saved* saved, const fno_workspace* ws, int batch,
                      int act_dtype, void* stream);

/* Backward of the above given dL/dpreds (float32 [B][2][64][64]); fills `grads`. */
int fno_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                 const float* case_params, const float* dpreds, const fno_train_saved* saved,
                 const fno_grads* grads, const fno_bwd_scratch* scratch, const fno_workspace* ws, int batch,
                 int act_dtype, void* stream);
/* Same backward, also differentiating w.r.t. the input frame and the case parameters (unrolled training through
 * rollouts, sensitivities / inverse problems with a frozen model; what autograd gives the reference when `inputs` or
 * `case_params` require grad, fno2d.py:195-217):
 *   d_inputs[b][c][h][w] = sum_o fc0_w[o][c] dL/da0[b][o][h][w]               c = 0 (u), 1 (v)
 *   d_case_params[b][j]  = sum_o fc0_w[o][5+j] sum_{h,w} dL/da0[b][o][h][w]
 * where a0 is the lift output (a bf16-stored a0 is differentiated straight through).  Both are overwritten and
 * bit-reproducible (fixed-order reductions, no atomics).  grads = NULL skips every parameter-gradient launch (data-only
 * backward, e.g. a frozen model); otherwise `grads` is filled as by fno_backward, and with d_inputs and d_case_params
 * both NULL the launches are exactly fno_backward's.  At least one of grads, d_inputs, d_case_params must be non-NULL;
 * d_inputs must be 16-byte aligned. */
int fno_backward_inputs(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                        const float* case_params, const float* dpreds, const fno_train_saved* saved,
                        const fno_grads* grads,        /* NULL: no parameter gradients (data-only backward) */
                        const fno_bwd_scratch* scratch, const fno_workspace* ws,
                        float* d_inputs,               /* [B][2][64][64] or NULL */
                        float* d_case_params,          /* [B][p] or NULL (must be NULL or unused when p == 0) */
                        int batch, int act_dtype, void* stream);

/* Training through a K-step rollout (backpropagation through time) with memory that does not grow with K beyond the
 * frames.  Frames are float32 [B][2][64][64]; preds_seq and dpreds_seq are [K][B][2][64][64].
 * fno_rollout_forward_train: K chained fno_forward_train calls, step s fed the (masked) prediction of step s-1, writing
 * preds_seq; `saved` is reused by every step (on return it holds step K-1's activations).  Its predictions are those of
 * K chained fno_forward_train calls, bit for bit.
 * fno_rollout_backward: the whole backward of that rollout in one call, for L = sum_s <dpreds_seq[s], preds_seq[s]>.  It
 * sweeps s = K-1 .. 0; each step recomputes step s's saved set from its input frame (`inputs` or preds_seq[s-1]) with
 * the training forward's kernels, then runs step s's backward with upstream gradient dpreds_seq[s] + carry, where carry
 * = dL/d(frame fed to step s+1).  The lift's data adjoint writes fc0[:, 0:2]^T dL/da0 + dpreds_seq[s-1] straight into
 * `carry` (float32 [B][2][64][64], its own buffer, used when K > 1).  grads (parameter gradients, summed over the steps),
 * d_inputs (dL/dinputs) and d_case_params (summed over the steps) are overwritten; each may be NULL, not all three.
 * Bit-reproducible (fixed-order reductions, no atomics); with K = 1 the results equal fno_forward_train +
 * fno_backward_inputs bit for bit.  d_inputs, carry and dpreds_seq must be 16-byte aligned.  steps < 1 -> status 1. */
int fno_rollout_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                              float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws, int batch,
                              int act_dtype, void* stream);
int fno_rollout_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                         const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                         const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                         const fno_workspace* ws, float* carry, float* d_inputs, float* d_case_params, int batch, int act_dtype,
                         void* stream);

/* Rollout evaluation on the device (SURVEY.md 8f.1; reference src/test_multistep.py:73-83,153-177 get_metrics on the
 * masked u channel, three .item() syncs per step and case there).  preds_seq [S][B][2][64][64], label_u and mask
 * [S][B][64][64]; sums [S][B][3] = (sum (p-l)^2, sum l^2, sum |p-l|) with p, l multiplied by mask. */
int fno_multistep_metrics(const float* preds_seq, const float* label_u, const float* mask, float* sums, int steps,
                          int batch, void* stream);

/* SURVEY.md 8f.2: one training batch gathered on the device from resident frames -- replaces DataLoader indexing +
 * collate_fn (reference src/train_auto.py:33-58: stack, channel slices, case-parameter dict loop, four .cuda() copies).
 * frames_in / frames_out: [N][3][64][64] (u, v, mask) as the dataset holds them (src/dataset/cavity.py:326-331), float32
 * (frame_dtype = FNO_ACT_F32) or bfloat16 (FNO_ACT_BF16); case_table [n_cases][p]; case_ids [N] int32; idx [n_idx] int64.
 * Outputs (float32): inputs [n][2][64][64], label [n][2][64][64], mask [n][1][64][64], case_params [n][p]. */
int fno_gather_batch(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                     const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                     float* mask, float* case_params, void* stream);

/* ---- the rest of a training step (reference src/train_auto.py:233-260) ------------------------------------- */

/* MseLoss.forward (reference src/models/loss.py:22-37) over n = preds.numel() float32 elements, one launch:
 * out[0..4] = mse, rmse, mae, nmse (= mse / mean(labels^2)), mean(labels^2).  scratch: fno_loss_scratch_bytes()
 * bytes, zero-initialised once by the caller (the kernel leaves it zeroed).  Deterministic. */
size_t fno_loss_scratch_bytes(void);
int fno_loss_fwd(const float* preds, const float* labels, size_t n, void* scratch, float* out, void* stream);
/* dpreds[i] = d(sum_j gout[j] * out[j]) / dpreds[i], gout = upstream gradients of (mse, rmse, mae, nmse);
 * `fwd` is the out[] of the matching fno_loss_fwd call. */
int fno_loss_bwd(const float* preds, const float* labels, const float* fwd, const float* gout, float* dpreds, size_t n,
                 void* stream);

/* torch.optim.Adam.step (train_auto.py:213,256; no amsgrad, maximize=False) for up to FNO_ADAM_MAX_TENSORS parameter
 * tensors in ONE launch.  Every array holds float32 views (a complex64 tensor is 2*numel floats, as
 * torch.view_as_real presents it to Adam); n[i] = number of floats.  `step` is the 1-based step count. */
#define FNO_ADAM_MAX_TENSORS 32
typedef struct fno_adam_tensors {
  int32_t count;
  void* param[FNO_ADAM_MAX_TENSORS];
  const void* grad[FNO_ADAM_MAX_TENSORS];
  void* exp_avg[FNO_ADAM_MAX_TENSORS];
  void* exp_avg_sq[FNO_ADAM_MAX_TENSORS];
  int64_t n[FNO_ADAM_MAX_TENSORS];
} fno_adam_tensors;
int fno_adam_step(const fno_adam_tensors* t, float lr, float beta1, float beta2, float eps, float weight_decay,
                  int64_t step, void* stream);

/* ---- one training step replayed from a CUDA graph, step after step (cfdbench_b200.train_auto) --------------------
 * What changes from step to step is read on the device through a step cursor `cursor` (one int32 in device memory,
 * reset by the caller at the start of an epoch and advanced by fno_train_log_step): the step's sample indices, Adam's
 * coefficients and the row of the step's losses.  Every entry point checks its arguments before any device work
 * (status 1 with a fno_last_error() message); a cursor that would read or write outside a table makes the launch write
 * nothing. */
/* idx_out[i] = perm[cursor * stride + i] for i < batch (int64 indices); nothing is written when
 * cursor * stride + batch > n_perm.  batch <= stride and batch <= n_perm. */
int fno_train_stage_indices(const int64_t* perm, int64_t n_perm, int stride, int batch, const int32_t* cursor,
                            int64_t* idx_out, void* stream);
/* fno_adam_step with (step_size, inv_bc2_sqrt) = (coef[2c], coef[2c + 1]), c = *cursor, read on the device; nothing is
 * written when c is outside 0..n_coef-1.  coef: 8-byte aligned float32 [n_coef][2], as fno_adam_coefficients fills it. */
int fno_adam_step_dev(const fno_adam_tensors* t, const float* coef, int n_coef, const int32_t* cursor, float beta1,
                      float beta2, float eps, float weight_decay, void* stream);
/* Host function: host_out[2i], host_out[2i + 1] = the step size lr / (1 - beta1^s) and 1 / sqrt(1 - beta2^s) of step
 * s = first_step + i, i < n, with exactly the arithmetic fno_adam_step uses (double, then float). */
int fno_adam_coefficients(float lr, float beta1, float beta2, int64_t first_step, int n, float* host_out);
/* log[c][0..4] = loss_out[0..4] (fno_loss_fwd's five scalars), c = *cursor, then ++*cursor; nothing is written when c is
 * outside 0..n_log-1. */
int fno_train_log_step(const float* loss_out, float* log, int n_log, int32_t* cursor, void* stream);

/* ---- gradient-norm clipping and an EMA of the weights (FusedAdam(max_grad_norm=..., ema_decay=...), train_auto) -----
 * torch.nn.utils.clip_grad_norm_(params, max_norm) followed by torch.optim.Adam.step, and diffusers' EMAModel.step after
 * it, fused into the Adam launch.  Argument checks come before any device work (status 1). */
/* The global norm: out[0] = ||g||_2 over the gradients of every entry of tables[0..n_tables-1] (the grad and n fields;
 * complex gradients as their real pairs, as torch counts them), out[1] = clip_grad_norm_'s coefficient
 * min(1, max_norm / (out[0] + 1e-6)) in float32 (evaluated as torch does, reciprocal(out[0] + 1e-6) * max_norm; a NaN
 * norm gives a NaN coefficient, an infinite norm 0).  The squares are summed in float64 by a fixed grid with per-block
 * partials and an in-order final sum (no float atomics), so the result is bit-reproducible; the norm is the float32
 * rounding of the square root.  With log != NULL also log[c] = out[0] for c = *cursor when 0 <= c < n_log (the step's row,
 * as fno_train_log_step picks it; the cursor is not advanced).  out: float32 [2] in device memory.  scratch:
 * fno_grad_norm_scratch_bytes() bytes, 8-byte aligned, zero-initialised once by the caller (the kernel leaves it zeroed);
 * one scratch buffer serves one stream at a time.  No host synchronisation; can be captured into a graph.  Status 1 for
 * n_tables outside 1..FNO_GRAD_NORM_MAX_TABLES, a bad table, max_norm not finite and > 0, or a null out / scratch
 * (or cursor, with log). */
#define FNO_GRAD_NORM_MAX_TABLES 8
size_t fno_grad_norm_scratch_bytes(void);
int fno_grad_norm(const fno_adam_tensors* tables, int n_tables, float max_norm, float* out, void* scratch, float* log,
                  int n_log, const int32_t* cursor, void* stream);
/* fno_adam_step with two optional additions, each selected by a non-NULL argument (with both NULL it is fno_adam_step):
 *   clip_coef (device float32, e.g. fno_grad_norm's out + 1): every gradient is read as g * (*clip_coef) before the
 *     weight decay -- clip_grad_norm_ before optimizer.step();
 *   ema (host array of t->count device pointers, ema[i] holding n[i] float32 like param[i]): after the update,
 *     ema[i] = fmaf(-d, p_new - ema[i], p_new) with d = min(ema_decay, 1 - step^(-3/4)) computed in double and rounded
 *     to float32 (fno_ema_decays), diffusers' EMAModel with use_ema_warmup, inv_gamma 1, power 3/4.  d = 0 at step 1, so
 *     the EMA then equals the weights.  ema_decay in [0, 1). */
int fno_adam_step_ex(const fno_adam_tensors* t, float lr, float beta1, float beta2, float eps, float weight_decay,
                     int64_t step, const float* clip_coef, void* const* ema, double ema_decay, void* stream);
/* fno_adam_step_dev with the same additions; the EMA decay is ema_decay_tab[c] (device float32 [n_coef], as
 * fno_ema_decays fills it) for c = *cursor, read on the device.  ema_decay_tab is required with ema and ignored without. */
int fno_adam_step_dev_ex(const fno_adam_tensors* t, const float* coef, int n_coef, const int32_t* cursor, float beta1,
                         float beta2, float eps, float weight_decay, const float* clip_coef, void* const* ema,
                         const float* ema_decay_tab, void* stream);
/* Host function: host_out[i] = the EMA decay fno_adam_step_ex uses at step first_step + i, i < n. */
int fno_ema_decays(double ema_decay, int64_t first_step, int n, float* host_out);

/* ---- training through K-step rollouts (cfdbench_b200.train_auto with rollout_steps = K) --------------------------
 * A dataset holds a case's samples contiguously with inputs = frames[:-s], labels = frames[s:] (s = time_step_size), so
 * the k-th target of the window that starts at sample j is labels[j + k s].  Every entry point checks its arguments before
 * any device work (status 1; a grid outside 24..128 returns 3); steps <= 32765. */
/* fno_gather_batch for the window starts idx, plus labels_seq [steps][n][2][64][64] float32:
 * labels_seq[k][b] = frames_out[idx[b] + k s][0:2] * frames_in[idx[b]][2] (one float32 multiply: label * mask).  inputs,
 * label, mask and case_params are fno_gather_batch's, bit for bit; label may be NULL (not written).  A window with
 * idx[b] + (steps - 1) s >= n_frames (the split's sample count) is not read and none of sample b's outputs are written. */
int fno_gather_window(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                      const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                      float* mask, float* case_params, int steps, int time_step_size, int64_t n_frames, float* labels_seq,
                      void* stream);
/* MseLoss of each step of a rollout and their mean, one launch: preds_seq / labels_seq [steps][n] float32 (n elements per
 * step, no alignment requirement).  out[k][0..4] = fno_loss_fwd's five scalars of step k, bit for bit (the same
 * reduction order); out[steps][c] = (out[0][c] + ... + out[steps-1][c]) * (1/steps), a left-to-right float32 sum times
 * the float32 reciprocal of steps, as `sum(...) / steps` computes it on 0-dim CUDA tensors.  scratch:
 * fno_loss_seq_scratch_bytes(steps) bytes, zero-initialised once by the caller (the kernel leaves it zeroed). */
size_t fno_loss_seq_scratch_bytes(int steps);
int fno_loss_seq_fwd(const float* preds_seq, const float* labels_seq, size_t n, int steps, void* scratch, float* out,
                     void* stream);
/* dpreds_seq[k] = fno_loss_bwd(preds_k, labels_k, fwd[k], gout * (1/steps)), bit for bit: gout = the upstream gradients
 * of the aggregate row's (mse, rmse, mae, nmse); fwd = the out[] of the matching fno_loss_seq_fwd call. */
int fno_loss_seq_bwd(const float* preds_seq, const float* labels_seq, const float* fwd, const float* gout, float* dpreds_seq,
                     size_t n, int steps, void* stream);

/* ---- training noise (cfdbench_b200.train_auto with input_noise_std > 0, DeviceFrames.batch(noise_std=...)) ----------
 * In place on n gathered input frames inputs [n][2][h][w] float32 with their masks mask [n][1][h][w]:
 *   inputs[b][c][y][x] = fmaf(std * z, mask[b][0][y][x], inputs[b][c][y][x])   where mask != 0 (other cells not written)
 * z is a standard normal and a pure function of (seed, step, j = idx[b], e), e = c h w + y w + x the element's index in
 * the sample's flattened (2, h, w) frame: (x0, x1, x2, x3) = Philox4x32-10(counter = (q, j, step & 0xffffffff,
 * step >> 32), key = (seed & 0xffffffff, seed >> 32)) for the quad q = e / 4 (the last quad is partial when h w is odd),
 * u_i = x_i 2^-32 + 2^-33 in float32, r = sqrtf(-2 logf(u0)), (z0, z1) = r (cospif(2 u1), sinpif(2 u1)), and (z2, z3)
 * likewise from (x2, x3); element e takes z_{e mod 4}.  step = *step_base + *step_offset (int64 + int32, both in device
 * memory, read when the kernel runs; step_offset may be NULL for 0), so a captured launch sees each replay's step.
 * 64x64 or any grid with 24 <= h, w <= 128; inputs and mask need only 4-byte alignment.  Status 3 for a grid outside
 * the range; status 1 for a null pointer (other than step_offset), n <= 0 or a negative or non-finite std. */
int fno_add_input_noise(float* inputs, const float* mask, const int64_t* idx, int n, int h, int w_, float std, uint64_t seed,
                        const int64_t* step_base, const int32_t* step_offset, void* stream);
/* Noise streams: the same noise with counter.x = q + (noise_stream << 16) instead of q, 0 <= noise_stream < 2^16.  Since
 * q < 2 * 128 * 128 / 4 = 2^13, no two streams share a counter, and stream 0 is fno_add_input_noise's noise bit for bit.
 * Out of place: out[b][c][y][x] = fmaf(std * z, mask[b][0][y][x], in[b][c][y][x]) where mask != 0, = in[b][c][y][x]
 * elsewhere; out may equal in.  Arguments and status codes as fno_add_input_noise (in, out: float32 [n][2][h][w]); also
 * status 1 for noise_stream outside 0 .. 2^16 - 1. */
#define FNO_NOISE_STREAMS 65536
int fno_add_input_noise_stream(const float* in, float* out, const float* mask, const int64_t* idx, int n, int h, int w_,
                               float std, uint64_t seed, const int64_t* step_base, const int32_t* step_offset,
                               int noise_stream, void* stream);

/* ---- noise on every step of a rollout (train_auto(noise_every_step=True), Fno2d.rollout(noise=...)) ---------------
 * The *_noise rollout drivers below take a noise descriptor and a fed-frames buffer `fed` [steps][B][2][H][W] float32 next
 * to preds_seq.  Call step s normally reads the frame x_s (inputs for s = 0, else preds_seq[s-1]); with stream
 * k = k0 + s >= 1 it reads fed[s] = fno_add_input_noise_stream(x_s, stream k) instead, which the forward drivers write
 * (one launch per such step) and the backward driver reads for its recomputation and the fc0 weight gradient (it
 * draws no noise: of the descriptor it reads only k0, the other fields are only checked).  Before its first launch a
 * forward driver also refuses what its per-step forward would refuse (status 1, or 3 for n_layers).  Stream 0
 * (a step 0 with k0 = 0) is never applied: the start frame's noise is the gather's (fno_add_input_noise, stream 0), so
 * fed[0] is then unused.  Full BPTT and a pushforward prefix pass k0 = 0, a trained tail after K - G prefix steps
 * k0 = K - G.  Predictions stay clean; dfed[s] / dx_s = I, so the gradients w.r.t. the frames flow as without noise.
 * The step is read on the device (*step_base + *step_offset) when each launch runs.  Every other argument is as in the
 * driver without noise; status 1 (before any device work) for a null descriptor, fed, idx or step_base, a negative or
 * non-finite std, k0 < 0 or k0 + steps > 2^16. */
typedef struct fno_noise {
  float std;
  uint64_t seed;
  const int64_t* idx;          /* [B] dataset index of each window start */
  const int64_t* step_base;    /* device int64 */
  const int32_t* step_offset;  /* device int32, or NULL for 0 */
  int32_t k0;                  /* the noise stream of the call's step 0 */
} fno_noise;
int fno_rollout_noise(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                      float* preds_seq, int steps, const fno_workspace* ws, const fno_noise* noise, float* fed, int batch,
                      int act_dtype, void* stream);
int fno_rollout_forward_train_noise(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                    float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws,
                                    const fno_noise* noise, float* fed, int batch, int act_dtype, void* stream);
int fno_rollout_backward_noise(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                               const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                               const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                               const fno_workspace* ws, const fno_noise* noise, const float* fed, float* carry,
                               float* d_inputs, float* d_case_params, int batch, int act_dtype, void* stream);

/* ---- teacher forcing of a rollout (train_auto(teacher_forcing=...), Fno2d.rollout(teacher=...)) -------------------
 * Scheduled sampling: rollout step s >= 1 of a window is fed the true frame of step s - 1 instead of the model's
 * prediction where a per-sample flag is set.
 * fno_teacher_flags: flags[s-1][i] = (u <= *prob) for s = 1 .. steps - 1 and i < batch (uint8 0 / 1), u = the uniform
 * of fno_add_input_noise's RNG, x0 2^-32 + 2^-33 in float32, from word x0 of Philox4x32-10(counter = (s, j,
 * step & 0xffffffff, step >> 32), key = (seed & 0xffffffff, seed >> 32)), j = idx[i]: a pure function of (seed, step, j,
 * s).  u lies in (0, 1], so *prob = 0 sets no flag and *prob = 1 every flag.  prob (float32) and step = *step_base +
 * *step_offset (step_offset may be NULL for 0) are read on the device when the kernel runs.  Status 1 for a null pointer
 * (other than step_offset), batch <= 0, steps < 2 or steps > 2^16.
 * The *_feed rollout drivers take a nullable noise descriptor (as the *_noise drivers) and a teacher descriptor:
 * frames [steps-1][B][2][H][W] float32 (the true frames, typically the masked window targets of steps 0 .. steps - 2)
 * and flags [steps-1][B].  The forward writes fed[s] = (flags[s-1][b] ? frames[s-1][b] : preds_seq[s-1][b]) for every
 * s >= 1 with one launch (plus the noise of stream k0 + s with a noise descriptor, as the *_noise drivers; a step 0 with
 * k0 >= 1 is fed as there) -- a choice of frame: a forced sample's fed frame never reads its prediction.  The backward
 * recomputes step s >= 1 from fed[s] and hands prediction s - 1 of a forced sample exactly dpreds_seq[s-1] (bit for bit;
 * nothing of step s's input gradient) and of any other sample fc0^T dL/da0 + dpreds_seq[s-1]; the parameter and
 * case-parameter gradients take every step's share as without a teacher.  Of the descriptor the backward reads only
 * flags (frames may be NULL there).  Every other argument and status code as the driver without a teacher; status 1
 * (before any device work) for a null teacher descriptor, fed or flags, or null frames in a forward driver. */
typedef struct fno_teacher {
  const float* frames;   /* [steps-1][B][2][H][W] */
  const uint8_t* flags;  /* [steps-1][B] */
} fno_teacher;
/* The status the teacher-forcing entry points return: 0, or the codes of the int-returning entry points above.  Their
 * pointer arguments' alignment contract is tested in tests/test_teacher_forcing_host.py: idx and step_base 8 bytes,
 * prob and step_offset 4; the *_feed drivers as the matching *_noise driver, teacher->frames 4 (float4 only where the
 * frames of a feed are 16-byte aligned), flags 1. */
typedef int fno_status;
fno_status fno_teacher_flags(const int64_t* idx, int batch, int steps, const float* prob, uint64_t seed, const int64_t* step_base,
                      const int32_t* step_offset, uint8_t* flags, void* stream);
fno_status fno_rollout_forward_train_feed(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                   float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws,
                                   const fno_noise* noise, const fno_teacher* teacher, float* fed, int batch, int act_dtype,
                                   void* stream);
fno_status fno_rollout_backward_feed(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                              const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                              const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                              const fno_workspace* ws, const fno_noise* noise, const fno_teacher* teacher, const float* fed,
                              float* carry, float* d_inputs, float* d_case_params, int batch, int act_dtype, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Grid-generic path: the same network on H x W frames with 24 <= H <= 128 and 24 <= W <= 128, e.g. CFDBench's
 * tube and dam problems (66 x 65, reference src/utils/autoregressive.py:24-26).  fp32 activation storage only (there is
 * no act_dtype argument); hidden 32, modes 12 x 12, in/out 2 channels and p <= 16 as above.  With H = W = 64 these entry
 * points run the generic kernels, not the 64 x 64 kernels above.  A grid outside the range returns FNO_ERR_UNSUPPORTED
 * (3) with a message.  They take the structs above with these layouts:
 *   frames / preds / d_inputs [B][2][H][W], mask [B][H][W]    float32, caller tensors: no alignment beyond 4 bytes needed
 *   activations, pre, d[]     [B][32][H*W]                     float32, fno_grid_act_bytes(B, H, W)
 *   modes (xm, ym, gm)        [288][B][32] complex64           as above; kxi 12..23 <-> kx H-12..H-1
 *   z                         [B][H][24][32] float32           fno_grid_z_bytes(B, H)
 *   dz1                       [min(B, FNO_BWD_CHUNK)][128][H*W] float32
 *   partials                  fno_grid_bwd_partials_bytes(H, W)
 *   fno_weights.gx / gy       H / W entries: float32(np.linspace(0, 1, n))
 * Twiddle tables are built in float64 on the host once per (device, H, W) on first use; fno_destroy releases them.
 * Gradients are bit-reproducible (per-CTA partial rows from a fixed number of CTAs, fixed-order reductions).
 * ------------------------------------------------------------------------------------------------- */
size_t fno_grid_act_bytes(int batch, int h, int w);
size_t fno_grid_z_bytes(int batch, int h);
size_t fno_grid_bwd_partials_bytes(int h, int w);
/* the stages, one launch each (same meaning as fno_lift_fwd .. fno_project_fwd) */
int fno_grid_lift_fwd(const float* inputs, const float* mask, const float* case_params, const fno_weights* w,
                      float* act_out, int batch, int h, int w_, void* stream);
int fno_grid_spectral_dft_fwd(const float* act_in, void* xm, int batch, int h, int w, float s0, float s1, void* stream);
int fno_grid_spectral_inv_kx(const void* ym, float* z, int batch, int h, int w, float s0, float s1, void* stream);
int fno_grid_block_out(int epilogue, const float* z, const float* act_in, const float* w0t, const float* bias, float* act_out,
                       float* pre_out, const float* pre_in, int batch, int h, int w, void* stream);
int fno_grid_project_fwd(const float* act_in, const float* mask, const fno_weights* w, float* preds, int batch, int h, int w_,
                         void* stream);
/* backward of fno_grid_project_fwd given dL/dpreds: dpre_out = dL/dpre of the last block (pre = its pre-activation),
 * and, when the four gradient pointers are set (all or none), the fc1 / fc2 gradients (overwritten).  dz1 and partials:
 * scratch as above. */
int fno_grid_project_bwd(const float* act_in, const float* dpreds, const float* mask, const float* pre, const fno_weights* w,
                         float* dpre_out, float* dz1, float* partials, float* g_fc1_w, float* g_fc1_b, float* g_fc2_w,
                         float* g_fc2_b, int batch, int h, int w_, void* stream);
/* fno_forward / fno_rollout / fno_forward_train on an H x W grid */
int fno_grid_forward(const fno_weights* w, const float* inputs, const float* mask, const float* case_params, float* preds,
                     const fno_workspace* ws, int batch, int h, int w_, void* stream);
int fno_grid_rollout(const fno_weights* w, const float* inputs, const float* mask, const float* case_params, float* preds_seq,
                     int steps, const fno_workspace* ws, int batch, int h, int w_, void* stream);
int fno_grid_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                           float* preds, const fno_train_saved* saved, const fno_workspace* ws, int batch, int h, int w_,
                           void* stream);
/* fno_backward_inputs on an H x W grid: grads = NULL gives the data-only backward */
int fno_grid_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                      const float* case_params, const float* dpreds, const fno_train_saved* saved, const fno_grads* grads,
                      const fno_bwd_scratch* scratch, const fno_workspace* ws, float* d_inputs, float* d_case_params,
                      int batch, int h, int w_, void* stream);
/* fno_rollout_forward_train / fno_rollout_backward on an H x W grid (frames, preds_seq, dpreds_seq and carry with H x W
 * planes; no alignment requirement) */
int fno_grid_rollout_forward_train(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                                   float* preds_seq, int steps, const fno_train_saved* saved, const fno_workspace* ws,
                                   int batch, int h, int w_, void* stream);
int fno_grid_rollout_backward(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                              const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                              const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                              const fno_workspace* ws, float* carry, float* d_inputs, float* d_case_params, int batch, int h,
                              int w_, void* stream);
/* the *_noise rollout drivers (above) on an H x W grid */
int fno_grid_rollout_noise(const fno_weights* w, const float* inputs, const float* mask, const float* case_params,
                           float* preds_seq, int steps, const fno_workspace* ws, const fno_noise* noise, float* fed,
                           int batch, int h, int w_, void* stream);
int fno_grid_rollout_forward_train_noise(const fno_weights* w, const float* inputs, const float* mask,
                                         const float* case_params, float* preds_seq, int steps, const fno_train_saved* saved,
                                         const fno_workspace* ws, const fno_noise* noise, float* fed, int batch, int h, int w_,
                                         void* stream);
int fno_grid_rollout_backward_noise(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                                    const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                                    const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                                    const fno_workspace* ws, const fno_noise* noise, const float* fed, float* carry,
                                    float* d_inputs, float* d_case_params, int batch, int h, int w_, void* stream);
/* the *_feed rollout drivers (above) on an H x W grid */
fno_status fno_grid_rollout_forward_train_feed(const fno_weights* w, const float* inputs, const float* mask,
                                        const float* case_params, float* preds_seq, int steps, const fno_train_saved* saved,
                                        const fno_workspace* ws, const fno_noise* noise, const fno_teacher* teacher, float* fed,
                                        int batch, int h, int w_, void* stream);
fno_status fno_grid_rollout_backward_feed(const fno_weights* w, const fno_weights_bwd* wb, const float* inputs, const float* mask,
                                   const float* case_params, const float* preds_seq, const float* dpreds_seq, int steps,
                                   const fno_train_saved* saved, const fno_grads* grads, const fno_bwd_scratch* scratch,
                                   const fno_workspace* ws, const fno_noise* noise, const fno_teacher* teacher,
                                   const float* fed, float* carry, float* d_inputs, float* d_case_params, int batch, int h,
                                   int w_, void* stream);
/* fno_multistep_metrics on an H x W grid: preds_seq [S][B][2][H][W], label_u and mask [S][B][H][W]; sums [S][B][3] as
 * there (sums over the H*W pixels).  One CTA per (step, case) plane, fixed-order reduction: bit-reproducible.
 * steps <= 65535. */
int fno_grid_multistep_metrics(const float* preds_seq, const float* label_u, const float* mask, float* sums, int steps,
                               int batch, int h, int w_, void* stream);
/* fno_gather_batch on an H x W grid: frames_in / frames_out [N][3][H][W] float32 or bfloat16; outputs (float32)
 * inputs [n][2][H][W], label [n][2][H][W], mask [n][1][H][W], case_params [n][p]. */
int fno_grid_gather_batch(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                          const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                          float* mask, float* case_params, int h, int w_, void* stream);
/* fno_gather_window on an H x W grid (frames_in / frames_out [N][3][H][W], labels_seq [steps][n][2][H][W]) */
int fno_grid_gather_window(const void* frames_in, const void* frames_out, const float* case_table, const int32_t* case_ids,
                           const int64_t* idx, int n_idx, int n_case_params, int frame_dtype, float* inputs, float* label,
                           float* mask, float* case_params, int steps, int time_step_size, int64_t n_frames,
                           float* labels_seq, int h, int w_, void* stream);

/* Rollout metrics of the S-step windows of a device-resident split (cfdbench_b200.evaluate_rollout_auto), without
 * gathering the targets: frames_in / frames_out [N][3][64][64] (u, v, mask; n_frames = N) float32 (frame_dtype =
 * FNO_ACT_F32) or bfloat16 (FNO_ACT_BF16), starts [B] int64 window starts, preds_seq [S][B][2][64][64] float32 (the
 * inference rollout from the start samples).  With j = starts[b], m = frames_in[j][2] and s = time_step_size:
 *   sums[k][b] = (sum (p-l)^2, sum l^2, sum |p-l|),  p = preds_seq[k][b][0] * m,  l = frames_out[j + k s][0] * m,
 * equal bit for bit to fno_multistep_metrics on label_u[k][b] = frames_out[j + k s][0], mask[k][b] = m.  A window with
 * j < 0 or j + (S - 1) s >= n_frames is not read and its sums are not written.  One CTA per (step, window), fixed-order
 * reduction: bit-reproducible.  preds_seq must be 16-byte aligned, the frames 16-byte (fp32) or 8-byte (bf16) aligned.
 * A null pointer, steps outside 1..65535, batch, time_step_size or n_frames < 1 or a bad frame_dtype returns 1 before any
 * device work. */
int fno_window_metrics(const float* preds_seq, const void* frames_in, const void* frames_out, const int64_t* starts,
                       int steps, int batch, int time_step_size, int64_t n_frames, int frame_dtype, float* sums,
                       void* stream);
/* fno_window_metrics on an H x W grid (frames [N][3][H][W], preds_seq [S][B][2][H][W]; no alignment beyond the element
 * needed).  A grid outside 24..128 returns 3. */
int fno_grid_window_metrics(const float* preds_seq, const void* frames_in, const void* frames_out, const int64_t* starts,
                            int steps, int batch, int time_step_size, int64_t n_frames, int frame_dtype, float* sums, int h,
                            int w_, void* stream);

/* Single-step evaluation (reference src/train_auto.py:61-148, `evaluate`, which synchronises 2 x (number of scores)
 * times per batch): the per-sample sums its scores are made of, for any grid 24 <= H, W <= 128 (64 x 64 included).
 * preds, label, inputs [B][2][H][W], mask [B][1][H][W], float32 caller tensors (no alignment beyond 4 bytes needed);
 * preds as the model returns them (already masked).  sums [B][6]:
 *   0: sum (preds - label*mask)^2   1: sum |preds - label*mask|   2: sum (label*mask)^2      both channels, H*W pixels
 *   3: sum (inputs_u - label_u)^2   4: sum |inputs_u - label_u|   5: sum label_u^2           channel 0, no mask
 * One CTA per sample, fixed-order reduction: bit-reproducible.  A grid outside the range returns 3, a null pointer or
 * batch <= 0 returns 1, both before any device work. */
int fno_eval_sums(const float* preds, const float* label, const float* mask, const float* inputs, float* sums, int batch,
                  int h, int w_, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CFDBENCH_B200_H_ */
