"""cfdbench_b200 -- H100-native (sm_90a) FNO hot path for CFDBench.

Public surface mirrors the reference's for this path:
    Fno2d, SpectralConv2d_fast, FnoBlock   (reference src/models/fno/fno2d.py)
    AutoCfdModel                           (reference src/models/base_model.py)
    MseLoss, loss_name_to_fn               (reference src/models/loss.py)
    infer_multistep                        (reference src/test_multistep.py infer, batched on the device)
    evaluate_auto                          (reference src/train_auto.py evaluate, batched on the device)
    evaluate_rollout_auto                  (a split's S-step rollout error, on the device; train_auto's
                                            dev_rollout_steps=S selects checkpoints by it)
    train_auto                             (reference src/train_auto.py train, steps replayed from CUDA graphs;
                                            rollout_steps=K trains through K-step rollouts)
    unroll_lengths                         (the per-step prefix lengths of train_auto(random_unroll=True))
    rollout_windows                        (the valid K-step window starts of a split)
    RolloutNoise, add_input_noise          (per-step input noise of Fno2d.rollout, and its eager form)
    TeacherForcing, teacher_forcing_flags  (teacher forcing of Fno2d.rollout, and its device-drawn flags)
"""
from .base_model import AutoCfdModel
from .loss import MseLoss, loss_name_to_fn

__all__ = ["AutoCfdModel", "MseLoss", "loss_name_to_fn", "Fno2d", "FnoBlock", "SpectralConv2d_fast", "FusedAdam", "DeviceFrames",
           "infer_multistep", "evaluate_auto", "evaluate_rollout_auto", "train_auto", "unroll_lengths",
           "rollout_windows", "RolloutNoise", "add_input_noise", "TeacherForcing", "teacher_forcing_flags"]


def __getattr__(name):  # lazy: importing the package must not require the native library
    if name in ("Fno2d", "FnoBlock", "SpectralConv2d_fast"):
        from . import fno2d
        return getattr(fno2d, name)
    if name == "FusedAdam":
        from .optim import FusedAdam
        return FusedAdam
    if name == "DeviceFrames":
        from .data import DeviceFrames
        return DeviceFrames
    if name == "infer_multistep":
        from .metrics import infer_multistep
        return infer_multistep
    if name == "evaluate_auto":
        from .metrics import evaluate_auto
        return evaluate_auto
    if name == "evaluate_rollout_auto":
        from .metrics import evaluate_rollout_auto
        return evaluate_rollout_auto
    if name in ("rollout_windows", "RolloutNoise", "add_input_noise", "TeacherForcing", "teacher_forcing_flags"):
        from . import data
        return getattr(data, name)
    if name in ("train_auto", "unroll_lengths"):
        from . import train
        return getattr(train, name)
    raise AttributeError(name)
