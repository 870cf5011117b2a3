"""FusedAdam: torch.optim.Adam's update (reference src/train_auto.py:213: Adam(model.parameters(), lr), betas
(0.9, 0.999), eps 1e-8, weight_decay 0, no amsgrad) for every parameter tensor of the model in ONE kernel launch
(`fno_adam_step`).  Complex parameters are updated as pairs of reals, exactly as torch.optim.Adam treats them
(torch.view_as_real).  State keys match torch's ("step", "exp_avg", "exp_avg_sq"), so `state_dict()` round-trips
with the stock optimizer.  An opt-in: the reference script builds its own torch.optim.Adam, which keeps working.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def _real_view(t: torch.Tensor) -> torch.Tensor:
    return torch.view_as_real(t) if t.is_complex() else t


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0):
        if lr < 0 or eps < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1) or weight_decay < 0:
            raise ValueError("invalid Adam hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))

    def init_state(self, p: torch.Tensor) -> dict:
        """The state of parameter `p`, created as torch.optim.Adam creates it on its first step when it is empty."""
        st = self.state[p]
        if not st:
            st["step"] = torch.tensor(0.0)
            st["exp_avg"] = torch.zeros_like(p)
            st["exp_avg_sq"] = torch.zeros_like(p)
        return st

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = _lib.load()
        for group in self.param_groups:
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            dev = ps[0].device
            if dev.type != "cuda":
                raise _lib.FnoNativeError("FusedAdam needs CUDA parameters (there is no CPU path)")
            step = None
            keep = []  # contiguous gradient copies must outlive the asynchronous launch
            for i0 in range(0, len(ps), _lib.ADAM_MAX_TENSORS):
                chunk = ps[i0:i0 + _lib.ADAM_MAX_TENSORS]
                t = _lib.FnoAdamTensors()
                t.count = len(chunk)
                for i, p in enumerate(chunk):
                    if p.dtype not in (torch.float32, torch.complex64) or not p.is_contiguous() or p.device != dev:
                        raise _lib.FnoNativeError("FusedAdam: parameters must be contiguous float32/complex64 on one device")
                    st = self.init_state(p)
                    st["step"] += 1
                    s = int(st["step"].item())
                    if step is None:
                        step = s
                    elif s != step:
                        raise _lib.FnoNativeError("FusedAdam: parameters of one group must share the step count")
                    g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                    keep.append(g)
                    t.param[i] = _real_view(p).data_ptr()
                    t.grad[i] = _real_view(g).data_ptr()
                    t.exp_avg[i] = _real_view(st["exp_avg"]).data_ptr()
                    t.exp_avg_sq[i] = _real_view(st["exp_avg_sq"]).data_ptr()
                    t.n[i] = p.numel() * (2 if p.is_complex() else 1)
                with torch.cuda.device(dev):
                    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
                    b1, b2 = group["betas"]
                    _lib.check(lib.fno_adam_step(C.byref(t), group["lr"], b1, b2, group["eps"], group["weight_decay"],
                                                 step, stream), "fno_adam_step")
            for g in keep:
                g.record_stream(torch.cuda.current_stream(dev))
            # the kernel wrote through raw pointers: tell autograd (and Fno2d's packed-weight cache, which is keyed on
            # the parameters' version counters) that the tensors changed
            for p in ps:
                torch.autograd.graph.increment_version(p)
        return loss
