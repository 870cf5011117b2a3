"""Mirror of the reference loss interface (reference src/models/loss.py:8-50).

`MseLoss.forward(preds, labels)` returns a dict of 0-dim tensors {mse, rmse, mae[, nmse]};
`get_score_names()` drives `train_auto.evaluate` (reference src/train_auto.py:75,93).
Each value stays on the device and supports `.item()` / `.backward()`.

CUDA tensors go through the native kernels (`fno_loss_fwd` / `fno_loss_bwd`: one launch each instead of the
reference's five reductions plus their autograd graph); host tensors -- the CPU-side tests of the interface -- use
the same formulas written with torch ops.
"""
from __future__ import annotations

import ctypes as C
from typing import List

import torch
from torch import Tensor, nn


class _NativeLoss(torch.autograd.Function):
    """(mse, rmse, mae, nmse) as one float32 vector; backward = fno_loss_bwd."""

    _scratch: dict = {}

    @staticmethod
    def forward(ctx, preds: Tensor, labels: Tensor) -> Tensor:
        from . import _lib
        lib = _lib.load()
        p = _lib.aligned(preds.detach().float())   # fno_loss_fwd reads both as float4
        l = _lib.aligned(labels.detach().float())
        if p.shape != l.shape:
            raise ValueError(f"preds {tuple(p.shape)} and labels {tuple(l.shape)} differ")
        dev = p.device
        out = torch.empty(5, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            key = (dev, stream.cuda_stream)  # the partial-sum table is reused call after call: one per stream
            scratch = _NativeLoss._scratch.get(key)
            if scratch is None:
                scratch = torch.zeros(lib.fno_loss_scratch_bytes(), dtype=torch.uint8, device=dev)
                _NativeLoss._scratch[key] = scratch
            st = C.c_void_p(stream.cuda_stream)
            _lib.check(lib.fno_loss_fwd(p.data_ptr(), l.data_ptr(), p.numel(), scratch.data_ptr(), out.data_ptr(), st),
                       "fno_loss_fwd")
        ctx.save_for_backward(p, l, out)
        return out[:4]

    @staticmethod
    def backward(ctx, gout: Tensor):
        from . import _lib
        lib = _lib.load()
        p, l, out = ctx.saved_tensors
        g = gout.contiguous().float()
        dp = torch.empty_like(p)
        with torch.cuda.device(p.device):
            st = C.c_void_p(torch.cuda.current_stream(p.device).cuda_stream)
            _lib.check(lib.fno_loss_bwd(p.data_ptr(), l.data_ptr(), out.data_ptr(), g.data_ptr(), dp.data_ptr(),
                                        p.numel(), st), "fno_loss_bwd")
        return dp, None


class MseLoss(nn.Module):
    def __init__(self, normalize: bool, is_masked: bool = False):
        super().__init__()
        self.normalize = normalize
        self.is_masked = is_masked

    def get_score_names(self) -> List[str]:
        return ["mse", "rmse", "mae"] + (["nmse"] if self.normalize else [])

    def forward(self, preds: Tensor, labels: Tensor) -> dict:
        if preds.is_cuda:
            v = _NativeLoss.apply(preds, labels)
            out = {"mse": v[0], "rmse": v[1], "mae": v[2]}
            if self.normalize:
                out["nmse"] = v[3]
            return out
        diff = preds - labels
        mse = torch.mean(diff * diff)
        out = {"mse": mse, "rmse": torch.sqrt(mse), "mae": torch.mean(torch.abs(diff))}
        if self.normalize:
            out["nmse"] = mse / torch.mean(labels * labels)
        return out


def loss_name_to_fn(name: str, masked: bool = False) -> MseLoss:
    name = name.lower()
    if masked:
        raise NotImplementedError
    if name == "mse":
        return MseLoss(normalize=False)
    if name == "nmse":
        return MseLoss(normalize=True)
    raise NotImplementedError(name)
