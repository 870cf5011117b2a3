"""ctypes binding of libcfdbench_b200.so (C ABI in include/cfdbench_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcfdbench_b200.so")

FNO_MAX_LAYERS = 8
ABI_VERSION = 4
ACT_F32, ACT_BF16 = 0, 1
EPI_GELU, EPI_GELU_SAVE_PRE, EPI_MUL_DGELU, EPI_PLAIN = 0, 1, 2, 3


class FnoWeights(C.Structure):
    _fields_ = [
        ("n_layers", C.c_int32),
        ("n_case_params", C.c_int32),
        ("fc0_w", C.c_void_p),
        ("fc0_b", C.c_void_p),
        ("spec_wk", C.c_void_p * FNO_MAX_LAYERS),
        ("w0t", C.c_void_p * FNO_MAX_LAYERS),
        ("w0_b", C.c_void_p * FNO_MAX_LAYERS),
        ("fc1_w", C.c_void_p),
        ("fc1_b", C.c_void_p),
        ("fc2_w", C.c_void_p),
        ("fc2_b", C.c_void_p),
        ("gx", C.c_void_p),
        ("gy", C.c_void_p),
    ]


class FnoWorkspace(C.Structure):
    _fields_ = [("act", C.c_void_p * 2), ("xm", C.c_void_p), ("ym", C.c_void_p), ("z", C.c_void_p),
                ("ym_img", C.c_void_p)]


class FnoGrads(C.Structure):
    """Device pointers of the gradient buffers (all float32 / complex64, reference parameter layouts)."""
    _fields_ = [
        ("fc0_w", C.c_void_p),
        ("fc0_b", C.c_void_p),
        ("spec_w1", C.c_void_p * FNO_MAX_LAYERS),
        ("spec_w2", C.c_void_p * FNO_MAX_LAYERS),
        ("w0_w", C.c_void_p * FNO_MAX_LAYERS),
        ("w0_b", C.c_void_p * FNO_MAX_LAYERS),
        ("fc1_w", C.c_void_p),
        ("fc1_b", C.c_void_p),
        ("fc2_w", C.c_void_p),
        ("fc2_b", C.c_void_p),
    ]


class FnoTrainSaved(C.Structure):
    _fields_ = [("act", C.c_void_p * (FNO_MAX_LAYERS + 1)), ("pre", C.c_void_p * FNO_MAX_LAYERS),
                ("xm", C.c_void_p * FNO_MAX_LAYERS)]


class FnoWeightsBwd(C.Structure):
    _fields_ = [("spec_wkT", C.c_void_p * FNO_MAX_LAYERS), ("w0", C.c_void_p * FNO_MAX_LAYERS)]


class FnoBwdScratch(C.Structure):
    _fields_ = [("d", C.c_void_p * 2), ("dz1", C.c_void_p), ("gm", C.c_void_p), ("gwk", C.c_void_p),
                ("partials", C.c_void_p)]


BWD_CHUNK = 32
ADAM_MAX_TENSORS = 32
GRAD_NORM_MAX_TABLES = 8


class FnoAdamTensors(C.Structure):
    _fields_ = [("count", C.c_int32),
                ("param", C.c_void_p * ADAM_MAX_TENSORS), ("grad", C.c_void_p * ADAM_MAX_TENSORS),
                ("exp_avg", C.c_void_p * ADAM_MAX_TENSORS), ("exp_avg_sq", C.c_void_p * ADAM_MAX_TENSORS),
                ("n", C.c_int64 * ADAM_MAX_TENSORS)]


class FnoNoise(C.Structure):
    """fno_noise: the per-step noise of a rollout driver (include/cfdbench_b200.h)."""
    _fields_ = [("std", C.c_float), ("seed", C.c_uint64), ("idx", C.c_void_p), ("step_base", C.c_void_p),
                ("step_offset", C.c_void_p), ("k0", C.c_int32)]


class FnoTeacher(C.Structure):
    """fno_teacher: the true frames and per-sample flags of a teacher-forced rollout driver (include/cfdbench_b200.h)."""
    _fields_ = [("frames", C.c_void_p), ("flags", C.c_void_p)]


NOISE_STREAMS = 2 ** 16

_P = C.c_void_p
_I = C.c_int
_F = C.c_float

# name -> (restype, argtypes); every symbol declared in include/cfdbench_b200.h must be listed here
SIGNATURES = {
    "fno_version": (C.c_int, []),
    "fno_last_error": (C.c_char_p, []),
    "fno_destroy": (C.c_int, []),
    "fno_act_bytes": (C.c_size_t, [_I, _I]),
    "fno_modes_bytes": (C.c_size_t, [_I]),
    "fno_z_bytes": (C.c_size_t, [_I]),
    "fno_ym_image_bytes": (C.c_size_t, [_I]),
    "fno_bwd_partials_bytes": (C.c_size_t, []),
    "fno_mode_mix_image": (C.c_int, [_P, _P, _P, _I, _P]),
    "fno_block_fused": (C.c_int, [_P, _P, _P, _P, _P, _I, _P]),
    "fno_pack_spectral_weights": (C.c_int, [_P, _P, _P, _I, _P]),
    "fno_unpack_spectral_grads": (C.c_int, [_P, _P, _P, _P]),
    "fno_mix_operand_bytes": (C.c_size_t, []),
    "fno_pack_mix_operand": (C.c_int, [_P, _P, _P]),
    "fno_pack_mix_operand_from_weights": (C.c_int, [_P, _P, _P, _I, _P]),
    "fno_lift_fwd": (C.c_int, [_P, _P, _P, C.POINTER(FnoWeights), _P, _I, _I, _P]),
    "fno_spectral_dft_fwd": (C.c_int, [_P, _P, _I, _I, _F, _F, _P]),
    "fno_mode_mix": (C.c_int, [_P, _P, _P, _I, _P]),
    "fno_spectral_inv_kx": (C.c_int, [_P, _P, _I, _F, _F, _P]),
    "fno_block_out": (C.c_int, [_I, _P, _P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "fno_block_fwd": (C.c_int, [C.POINTER(FnoWeights), _I, _P, _P, _P, C.POINTER(FnoWorkspace), _I, _I, _P]),
    "fno_project_fwd": (C.c_int, [_P, _P, C.POINTER(FnoWeights), _P, _I, _I, _P]),
    "fno_forward": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, C.POINTER(FnoWorkspace), _I, _I, _P]),
    "fno_rollout": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoWorkspace), _I, _I, _P]),
    "fno_rollout_host": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoWorkspace), _P, _I, _I, _P]),
    "fno_rollout_host_scratch_bytes": (C.c_size_t, [_I, _I, _I]),
    "fno_multistep_metrics": (C.c_int, [_P, _P, _P, _P, _I, _I, _P]),
    "fno_gather_batch": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "fno_loss_scratch_bytes": (C.c_size_t, []),
    "fno_loss_fwd": (C.c_int, [_P, _P, C.c_size_t, _P, _P, _P]),
    "fno_loss_bwd": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, _P]),
    "fno_adam_step": (C.c_int, [C.POINTER(FnoAdamTensors), C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                C.c_int64, _P]),
    "fno_train_stage_indices": (C.c_int, [_P, C.c_int64, _I, _I, _P, _P, _P]),
    "fno_adam_step_dev": (C.c_int, [C.POINTER(FnoAdamTensors), _P, _I, _P, _F, _F, _F, _F, _P]),
    "fno_adam_coefficients": (C.c_int, [_F, _F, _F, C.c_int64, _I, _P]),
    "fno_train_log_step": (C.c_int, [_P, _P, _I, _P, _P]),
    # gradient-norm clipping and the EMA of the weights
    "fno_grad_norm_scratch_bytes": (C.c_size_t, []),
    "fno_grad_norm": (C.c_int, [C.POINTER(FnoAdamTensors), _I, _F, _P, _P, _P, _I, _P, _P]),
    "fno_adam_step_ex": (C.c_int, [C.POINTER(FnoAdamTensors), _F, _F, _F, _F, _F, C.c_int64, _P, C.POINTER(_P),
                                   C.c_double, _P]),
    "fno_adam_step_dev_ex": (C.c_int, [C.POINTER(FnoAdamTensors), _P, _I, _P, _F, _F, _F, _F, _P, C.POINTER(_P), _P, _P]),
    "fno_ema_decays": (C.c_int, [C.c_double, C.c_int64, _I, _P]),
    "fno_forward_train": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, C.POINTER(FnoTrainSaved),
                                    C.POINTER(FnoWorkspace), _I, _I, _P]),
    "fno_backward": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P,
                               C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                               C.POINTER(FnoWorkspace), _I, _I, _P]),
    "fno_backward_inputs": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P,
                                      C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                      C.POINTER(FnoWorkspace), _P, _P, _I, _I, _P]),
    "fno_rollout_forward_train": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoTrainSaved),
                                            C.POINTER(FnoWorkspace), _I, _I, _P]),
    "fno_rollout_backward": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P, _P, _I,
                                       C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                       C.POINTER(FnoWorkspace), _P, _P, _P, _I, _I, _P]),
    # grid-generic fp32 path (H, W in 24..128)
    "fno_grid_act_bytes": (C.c_size_t, [_I, _I, _I]),
    "fno_grid_z_bytes": (C.c_size_t, [_I, _I]),
    "fno_grid_bwd_partials_bytes": (C.c_size_t, [_I, _I]),
    "fno_grid_lift_fwd": (C.c_int, [_P, _P, _P, C.POINTER(FnoWeights), _P, _I, _I, _I, _P]),
    "fno_grid_spectral_dft_fwd": (C.c_int, [_P, _P, _I, _I, _I, _F, _F, _P]),
    "fno_grid_spectral_inv_kx": (C.c_int, [_P, _P, _I, _I, _I, _F, _F, _P]),
    "fno_grid_block_out": (C.c_int, [_I, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "fno_grid_project_fwd": (C.c_int, [_P, _P, C.POINTER(FnoWeights), _P, _I, _I, _I, _P]),
    "fno_grid_project_bwd": (C.c_int, [_P, _P, _P, _P, C.POINTER(FnoWeights), _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "fno_grid_forward": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, C.POINTER(FnoWorkspace), _I, _I, _I, _P]),
    "fno_grid_rollout": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoWorkspace), _I, _I, _I, _P]),
    "fno_grid_forward_train": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, C.POINTER(FnoTrainSaved),
                                         C.POINTER(FnoWorkspace), _I, _I, _I, _P]),
    "fno_grid_backward": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P,
                                    C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                    C.POINTER(FnoWorkspace), _P, _P, _I, _I, _I, _P]),
    "fno_grid_rollout_forward_train": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoTrainSaved),
                                                 C.POINTER(FnoWorkspace), _I, _I, _I, _P]),
    "fno_grid_rollout_backward": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P, _P, _I,
                                            C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                            C.POINTER(FnoWorkspace), _P, _P, _P, _I, _I, _I, _P]),
    "fno_grid_multistep_metrics": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "fno_grid_gather_batch": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _I, _I, _P]),
    "fno_eval_sums": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    # training through K-step rollouts
    "fno_gather_window": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _I, _I, C.c_int64, _P, _P]),
    "fno_grid_gather_window": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _I, _I, C.c_int64, _P, _I, _I,
                                         _P]),
    "fno_loss_seq_scratch_bytes": (C.c_size_t, [_I]),
    "fno_loss_seq_fwd": (C.c_int, [_P, _P, C.c_size_t, _I, _P, _P, _P]),
    "fno_loss_seq_bwd": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, _I, _P]),
    # rollout metrics of a split's windows
    "fno_window_metrics": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, C.c_int64, _I, _P, _P]),
    "fno_grid_window_metrics": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, C.c_int64, _I, _P, _I, _I, _P]),
    # training noise
    "fno_add_input_noise": (C.c_int, [_P, _P, _P, _I, _I, _I, _F, C.c_uint64, _P, _P, _P]),
    "fno_add_input_noise_stream": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _F, C.c_uint64, _P, _P, _I, _P]),
    # noise on every step of a rollout
    "fno_rollout_noise": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoWorkspace),
                                    C.POINTER(FnoNoise), _P, _I, _I, _P]),
    "fno_rollout_forward_train_noise": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoTrainSaved),
                                                  C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), _P, _I, _I, _P]),
    "fno_rollout_backward_noise": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P, _P, _I,
                                             C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                             C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), _P, _P, _P, _P, _I, _I, _P]),
    "fno_grid_rollout_noise": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoWorkspace),
                                         C.POINTER(FnoNoise), _P, _I, _I, _I, _P]),
    "fno_grid_rollout_forward_train_noise": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I,
                                                       C.POINTER(FnoTrainSaved), C.POINTER(FnoWorkspace),
                                                       C.POINTER(FnoNoise), _P, _I, _I, _I, _P]),
    "fno_grid_rollout_backward_noise": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P, _P, _I,
                                                  C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                                  C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), _P, _P, _P, _P, _I, _I,
                                                  _I, _P]),
    # teacher forcing of a rollout
    "fno_teacher_flags": (C.c_int, [_P, _I, _I, _P, C.c_uint64, _P, _P, _P, _P]),
    "fno_rollout_forward_train_feed": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoTrainSaved),
                                                 C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), C.POINTER(FnoTeacher), _P,
                                                 _I, _I, _P]),
    "fno_rollout_backward_feed": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P, _P, _I,
                                            C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                            C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), C.POINTER(FnoTeacher), _P, _P, _P,
                                            _P, _I, _I, _P]),
    "fno_grid_rollout_forward_train_feed": (C.c_int, [C.POINTER(FnoWeights), _P, _P, _P, _P, _I, C.POINTER(FnoTrainSaved),
                                                      C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), C.POINTER(FnoTeacher),
                                                      _P, _I, _I, _I, _P]),
    "fno_grid_rollout_backward_feed": (C.c_int, [C.POINTER(FnoWeights), C.POINTER(FnoWeightsBwd), _P, _P, _P, _P, _P, _I,
                                                 C.POINTER(FnoTrainSaved), C.POINTER(FnoGrads), C.POINTER(FnoBwdScratch),
                                                 C.POINTER(FnoWorkspace), C.POINTER(FnoNoise), C.POINTER(FnoTeacher), _P,
                                                 _P, _P, _P, _I, _I, _I, _P]),
}

GRID_MIN, GRID_MAX = 24, 128

_lib = None


class FnoNativeError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the native library once.  Raises FnoNativeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FnoNativeError(
            f"{LIB_PATH} is missing: build it with `python -m cfdbench_b200.build` "
            "(there is no CPU or PyTorch fallback for the FNO kernels)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.fno_version() != ABI_VERSION:
        raise FnoNativeError(f"ABI version mismatch: library reports {lib.fno_version()}, wrapper expects {ABI_VERSION}")
    _lib = lib
    return lib


def check(status: int, what: str) -> None:
    if status != 0:
        msg = load().fno_last_error()
        raise FnoNativeError(f"{what} failed with status {status}: {msg.decode() if msg else '?'}")


def aligned(t):
    """`t` as a contiguous tensor whose data pointer is 16-byte aligned: `t` itself when it already is, else a copy.

    The C ABI refuses a caller pointer that is less aligned than its kernels' widest access through it (16 bytes for the
    float4 / TMA reads of the 64x64 path).  A contiguous view can start at any element of its storage -- e.g.
    `flat[p * B:].view(B, 2, 64, 64)` of a staging buffer -- so the modules pass every caller tensor that reaches such a
    pointer through this: the ABI refuses, the module copies."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()
