"""FusedAdam: torch.optim.Adam's update (reference src/train_auto.py:213: Adam(model.parameters(), lr), betas
(0.9, 0.999), eps 1e-8, weight_decay 0, no amsgrad) for every parameter tensor of the model in ONE kernel launch
(`fno_adam_step_ex`).  Complex parameters are updated as pairs of reals, exactly as torch.optim.Adam treats them
(torch.view_as_real).  State keys match torch's ("step", "exp_avg", "exp_avg_sq"), so `state_dict()` round-trips
with the stock optimizer.  An opt-in: the reference script builds its own torch.optim.Adam, which keeps working.

Two opt-in safeguards run inside that launch:
- max_grad_norm: `torch.nn.utils.clip_grad_norm_(all parameters with a gradient, max_grad_norm)` before the update,
  one float64 norm launch (`fno_grad_norm`) over every param group; the pre-clip norm stays on the device as
  `last_grad_norm`.
- ema_decay: an exponential moving average of the weights in each parameter's state["ema"], diffusers' EMAModel with
  warmup (decay min(ema_decay, 1 - t^(-3/4)) at Adam's step t, inv_gamma 1, power 3/4); `copy_ema_to(module)` copies it
  into a module, as EMAModel.copy_to does.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers

import torch

from . import _lib


def _real_view(t: torch.Tensor) -> torch.Tensor:
    return torch.view_as_real(t) if t.is_complex() else t


def check_stabiliser_args(max_grad_norm, ema_decay):
    """(max_grad_norm, ema_decay) as floats or None; ValueError unless max_grad_norm is None or a finite real > 0 and
    ema_decay None or a real in [0, 1)."""
    def real(v):
        return isinstance(v, numbers.Real) and not isinstance(v, bool)
    if max_grad_norm is not None:
        if not real(max_grad_norm) or not math.isfinite(float(max_grad_norm)) or not float(max_grad_norm) > 0:
            raise ValueError(f"max_grad_norm must be None or a finite real number > 0, got {max_grad_norm!r}")
        max_grad_norm = float(max_grad_norm)
    if ema_decay is not None:
        if not real(ema_decay) or not 0 <= float(ema_decay) < 1:
            raise ValueError(f"ema_decay must be None or a real number in [0, 1), got {ema_decay!r}")
        ema_decay = float(ema_decay)
    return max_grad_norm, ema_decay


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 max_grad_norm=None, ema_decay=None):
        if lr < 0 or eps < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1) or weight_decay < 0:
            raise ValueError("invalid Adam hyper-parameter")
        self.max_grad_norm, self.ema_decay = check_stabiliser_args(max_grad_norm, ema_decay)
        self.last_grad_norm = None   # with max_grad_norm: the last step's pre-clip norm, a 0-dim device tensor
        self._norm_scratch = {}      # device -> the norm kernel's scratch
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))

    def init_state(self, p: torch.Tensor) -> dict:
        """The state of parameter `p`, created as torch.optim.Adam creates it on its first step when it is empty; with
        ema_decay also "ema", a copy of `p` before its first update."""
        st = self.state[p]
        if not st:
            st["step"] = torch.tensor(0.0)
            st["exp_avg"] = torch.zeros_like(p)
            st["exp_avg_sq"] = torch.zeros_like(p)
            if self.ema_decay is not None:
                st["ema"] = p.detach().clone()
        return st

    def norm_scratch(self, dev: torch.device) -> torch.Tensor:
        """The zeroed scratch of fno_grad_norm on `dev` (the kernel leaves it zeroed), one per optimizer and device."""
        s = self._norm_scratch.get(dev)
        if s is None:
            n = _lib.load().fno_grad_norm_scratch_bytes()
            s = self._norm_scratch[dev] = torch.zeros((n + 7) // 8, dtype=torch.float64, device=dev)
        return s

    @torch.no_grad()
    def copy_ema_to(self, module: torch.nn.Module) -> None:
        """Copy the EMA weights into `module`, whose parameters() list matches this optimizer's parameters in order (the
        model it trains, or another instance of it).  A parameter without an EMA (frozen: it never had a step) is copied
        as it is.  The copies bump the module's version counters, so a Fno2d rebuilds its packed weights."""
        if self.ema_decay is None:
            raise ValueError("copy_ema_to needs an optimizer built with ema_decay")
        src = [p for g in self.param_groups for p in g["params"]]
        dst = list(module.parameters())
        if len(src) != len(dst) or any(a.shape != b.shape or a.dtype != b.dtype for a, b in zip(src, dst)):
            raise ValueError("copy_ema_to: the module's parameters do not match the optimizer's")
        for a, b in zip(src, dst):
            st = self.state.get(a)
            b.copy_(st["ema"] if st and "ema" in st else a)

    @staticmethod
    def _tables(ps, grads, states=None, ema: bool = False) -> list:
        """The FnoAdamTensors tables of one update over the parameters `ps` with gradients `grads`, in order, up to
        ADAM_MAX_TENSORS entries each; complex tensors enter as pairs of reals.  With `states` (init_state's dicts) the
        entries also point at the moments (the norm reads only grad and n).  Each table's `ema` is the array of its
        entries' state["ema"] pointers when `ema`, else None."""
        out = []
        for i0 in range(0, len(ps), _lib.ADAM_MAX_TENSORS):
            t = _lib.FnoAdamTensors()
            t.count = min(_lib.ADAM_MAX_TENSORS, len(ps) - i0)
            for j in range(t.count):
                p, g = ps[i0 + j], grads[i0 + j]
                t.param[j] = _real_view(p).data_ptr()
                t.grad[j] = _real_view(g).data_ptr()
                t.n[j] = p.numel() * (2 if p.is_complex() else 1)
                if states is not None:
                    t.exp_avg[j] = _real_view(states[i0 + j]["exp_avg"]).data_ptr()
                    t.exp_avg_sq[j] = _real_view(states[i0 + j]["exp_avg_sq"]).data_ptr()
            t.ema = (C.c_void_p * t.count)(*[_real_view(st["ema"]).data_ptr() for st in states[i0:i0 + t.count]]) \
                if ema else None
            out.append(t)
        return out

    @torch.no_grad()
    def step(self, closure=None):
        """One Adam update of every parameter with a gradient.  Every group is validated and its step count advanced
        before the first launch, so a refused input launches nothing.  Then, with max_grad_norm, one fno_grad_norm over
        every group's gradients, and one fno_adam_step_ex per group and table (no clip coefficient and no EMA tensors
        without the options: the plain update)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = _lib.load()
        one_device = self.max_grad_norm is not None or self.ema_decay is not None   # the norm spans every group
        groups, dev = [], None
        for group in self.param_groups:
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            if dev is None or not one_device:
                dev = ps[0].device
                if dev.type != "cuda":
                    raise _lib.FnoNativeError("FusedAdam needs CUDA parameters (there is no CPU path)")
            step, states = None, []
            for p in ps:
                if p.dtype not in (torch.float32, torch.complex64) or not p.is_contiguous() or p.device != dev:
                    raise _lib.FnoNativeError("FusedAdam: parameters must be contiguous float32/complex64 on one device")
                st = self.init_state(p)
                st["step"] += 1
                s = int(st["step"].item())
                if step is None:
                    step = s
                elif s != step:
                    raise _lib.FnoNativeError("FusedAdam: parameters of one group must share the step count")
                states.append(st)
            # contiguous gradient copies must outlive the asynchronous launches
            grads = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ps]
            groups.append((group, dev, ps, grads, step, self._tables(ps, grads, states, self.ema_decay is not None)))
        if not groups:
            return loss
        clip = None
        if self.max_grad_norm is not None:
            tables = [t for *_, tabs in groups for t in tabs]
            if len(tables) > _lib.GRAD_NORM_MAX_TABLES:
                raise _lib.FnoNativeError(f"FusedAdam(max_grad_norm=...): at most "
                                          f"{_lib.GRAD_NORM_MAX_TABLES * _lib.ADAM_MAX_TENSORS} parameter tensors")
            with torch.cuda.device(dev):
                out = torch.empty(2, dtype=torch.float32, device=dev)   # norm, coefficient
                _lib.check(lib.fno_grad_norm((_lib.FnoAdamTensors * len(tables))(*tables), len(tables), self.max_grad_norm,
                                             out.data_ptr(), self.norm_scratch(dev).data_ptr(), None, 0, None,
                                             C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "fno_grad_norm")
            self.last_grad_norm = out[0]
            clip = out[1:].data_ptr()
        ema_decay = 0.0 if self.ema_decay is None else self.ema_decay
        for group, dev, ps, grads, step, tabs in groups:
            b1, b2 = group["betas"]
            with torch.cuda.device(dev):
                cur = torch.cuda.current_stream(dev)
                for t in tabs:
                    _lib.check(lib.fno_adam_step_ex(C.byref(t), group["lr"], b1, b2, group["eps"], group["weight_decay"],
                                                    step, clip, t.ema, ema_decay, C.c_void_p(cur.cuda_stream)),
                               "fno_adam_step_ex")
                for g in grads:
                    g.record_stream(cur)
            # the kernel wrote through raw pointers: tell autograd (and Fno2d's packed-weight cache, which is keyed on
            # the parameters' version counters) that the tensors changed
            for p in ps:
                torch.autograd.graph.increment_version(p)
        return loss
