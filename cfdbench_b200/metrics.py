"""Device-side rollout evaluation (SURVEY.md 8f.1).

`multistep_metrics` reproduces what `test_multistep.infer` reports (reference src/test_multistep.py:153-177):
for every rollout step, the mean over cases of `get_metrics(preds_u * mask, label_u * mask)`
(`mse`, `nmse = mse / mean(label^2)`, `mae`; reference :73-83) -- with ONE kernel launch and ONE device->host copy
instead of three `.item()` synchronisations per step and case.

`infer_multistep` replaces the whole of `test_multistep.infer` for an autoregressive model: the reference rolls out one
case at a time with B = 1 (`infer_case`, :102-132) and then synchronises three times per step and case; here the cases
run as one batched, graph-replayed rollout per chunk of at most `max_batch` cases, each followed by one metrics launch,
and the whole split makes one device->host copy.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib

HW = 64 * 64


def _check_grid(gh: int, gw: int) -> None:
    if not (_lib.GRID_MIN <= gh <= _lib.GRID_MAX and _lib.GRID_MIN <= gw <= _lib.GRID_MAX):
        raise ValueError(f"grid {gh}x{gw} is outside the supported range {_lib.GRID_MIN}..{_lib.GRID_MAX} in H and W")


def _launch_metrics(preds: Tensor, label_u: Tensor, mask: Tensor, sums: Tensor) -> None:
    """sums [S][B][3] (a contiguous float32 CUDA tensor or view) <- the per-plane sums of preds / label_u / mask, which
    must be contiguous float32 CUDA tensors of the shapes multistep_metrics checks."""
    s, b, _, gh, gw = preds.shape
    lib = _lib.load()
    with torch.cuda.device(preds.device):
        st = C.c_void_p(torch.cuda.current_stream(preds.device).cuda_stream)
        if (gh, gw) == (64, 64):
            _lib.check(lib.fno_multistep_metrics(preds.data_ptr(), label_u.data_ptr(), mask.data_ptr(), sums.data_ptr(),
                                                 s, b, st), "fno_multistep_metrics")
        else:
            _lib.check(lib.fno_grid_multistep_metrics(preds.data_ptr(), label_u.data_ptr(), mask.data_ptr(),
                                                      sums.data_ptr(), s, b, gh, gw, st), "fno_grid_multistep_metrics")


def _per_case(host: np.ndarray, hw: int) -> Dict[str, np.ndarray]:
    """(..., 3) float64 sums -> per-case mse, nmse, mae (reference get_metrics, :73-83)."""
    mse = host[..., 0] / hw
    return dict(mse=mse, nmse=mse / (host[..., 1] / hw), mae=host[..., 2] / hw)


def multistep_metrics(preds: Union[Tensor, Sequence[Tensor]], label_u: Tensor, mask: Tensor) -> List[Dict[str, float]]:
    """preds: (S,B,2,H,W) tensor or the list `generate_many` returns; label_u, mask: (S,B,H,W) CUDA tensors
    (the reference compares step s with frame s of the case, u channel only, using that frame's mask).  64x64 frames and
    any grid with 24 <= H, W <= 128 (the tube and dam problems' 66x65).
    Returns a list of S dicts {mse, nmse, mae}, each the mean over the B cases (as `combine_dicts` does)."""
    if not isinstance(preds, Tensor):
        preds = torch.stack(list(preds))
    if preds.dim() != 5 or preds.shape[2] != 2:
        raise ValueError(f"expected preds (S,B,2,H,W), got {tuple(preds.shape)}")
    s, b, _, gh, gw = preds.shape
    _check_grid(gh, gw)
    if tuple(label_u.shape) != (s, b, gh, gw) or tuple(mask.shape) != (s, b, gh, gw):
        raise ValueError(f"expected preds (S,B,2,H,W), label_u (S,B,H,W), mask (S,B,H,W); got {tuple(preds.shape)}, "
                         f"{tuple(label_u.shape)}, {tuple(mask.shape)}")
    if preds.device.type != "cuda":
        raise _lib.FnoNativeError("multistep_metrics has no CPU path: pass CUDA tensors")
    preds = preds.contiguous().float()
    label_u = label_u.to(preds.device).contiguous().float()
    mask = mask.to(preds.device).contiguous().float()
    sums = torch.empty(s, b, 3, dtype=torch.float32, device=preds.device)
    _launch_metrics(preds, label_u, mask, sums)
    host = sums.double().cpu()  # the only synchronisation
    per_case = _per_case(host.numpy(), gh * gw)
    return [{k: float(torch.from_numpy(v[i]).mean()) for k, v in per_case.items()} for i in range(s)]


def infer_multistep(model, all_features: Sequence[Union[Tensor, np.ndarray]], all_case_params: Sequence[Tensor],
                    infer_steps: int = 20, max_batch: int = 256) -> List[Dict[str, float]]:
    """What `test_multistep.infer(model, all_features, all_case_params, infer_steps)` returns for an autoregressive model
    (reference src/test_multistep.py:135-177): a list of `infer_steps` dicts {mse, nmse, mae}, each the mean over cases.

    all_features: one (T_c, 3, H, W) tensor or array per case (u, v, mask; any device), T_c >= infer_steps and one grid
    for all cases; all_case_params: one (p,) tensor per case.  Case c starts from features[c][0, :2] and rolls out with
    the mask features[c][0, 2] and all_case_params[c]; prediction s (0-based) is compared with frame s of the case (the
    reference's indexing), u channel only, both sides multiplied by frame s's mask.

    Cases run in chunks of at most `max_batch`: per chunk one `generate_many` (the graph-replayed rollout, no autograd)
    and one metrics launch into a device buffer for the whole split, which is copied to the host once at the end and
    reduced there in float64 over cases in index order.  Samples of a batch are computed independently, so the result
    does not depend on `max_batch`."""
    n = len(all_features)
    if n == 0 or len(all_case_params) != n:
        raise ValueError("all_features and all_case_params must be non-empty lists of the same length")
    if infer_steps < 1 or max_batch < 1:
        raise ValueError("infer_steps and max_batch must be positive")
    feats = [f if isinstance(f, Tensor) else torch.from_numpy(np.asarray(f)) for f in all_features]
    shape = tuple(feats[0].shape[1:])
    for c, f in enumerate(feats):
        if f.dim() != 4 or f.shape[1] != 3:
            raise ValueError(f"case {c}: expected (T, 3, H, W) frames (u, v, mask), got {tuple(f.shape)}")
        if tuple(f.shape[1:]) != shape:
            raise ValueError(f"case {c}: frames {tuple(f.shape[1:])} do not match case 0's {shape}: the cases of a split "
                             "must share one grid")
        if f.shape[0] < infer_steps:
            raise ValueError(f"case {c} has {f.shape[0]} frames, fewer than infer_steps={infer_steps}: pad it by repeating "
                             "its last frame, as test_multistep.main does")
    gh, gw = shape[1:]
    _check_grid(gh, gw)
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise _lib.FnoNativeError("infer_multistep has no CPU path: the model must be on a CUDA device")
    s = infer_steps
    sums = torch.empty(s * n * 3, dtype=torch.float32, device=dev)   # chunk k's (S, B_k, 3) block at offset S*lo*3
    with torch.no_grad():
        for lo in range(0, n, max_batch):
            hi = min(n, lo + max_batch)
            fr = torch.stack([f[:s].to(device=dev, dtype=torch.float32) for f in feats[lo:hi]])   # (B, S, 3, H, W)
            cp = torch.stack([p.to(device=dev, dtype=torch.float32).reshape(-1) for p in all_case_params[lo:hi]])
            preds = model.generate_many(inputs=fr[:, 0, :2], case_params=cp, mask=fr[:, 0, 2], steps=s)
            preds = torch.stack(preds)                             # (S, B, 2, H, W)
            label_u = fr[:, :, 0].transpose(0, 1).contiguous()     # (S, B, H, W): frame s of each case
            mask = fr[:, :, 2].transpose(0, 1).contiguous()
            _launch_metrics(preds, label_u, mask, sums[s * lo * 3:s * hi * 3])
    host = sums.double().cpu().numpy()   # the only synchronisation
    blocks = []
    for lo in range(0, n, max_batch):
        hi = min(n, lo + max_batch)
        blocks.append(host[s * lo * 3:s * hi * 3].reshape(s, hi - lo, 3))
    per_case = _per_case(np.concatenate(blocks, axis=1), gh * gw)   # (S, n) each
    return [{k: float(np.mean(v[i])) for k, v in per_case.items()} for i in range(s)]
