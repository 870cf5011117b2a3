"""Device-side rollout evaluation (SURVEY.md 8f.1).

`multistep_metrics` reproduces what `test_multistep.infer` reports (reference src/test_multistep.py:153-177):
for every rollout step, the mean over cases of `get_metrics(preds_u * mask, label_u * mask)`
(`mse`, `nmse = mse / mean(label^2)`, `mae`; reference :73-83) -- with ONE kernel launch and ONE device->host copy
instead of three `.item()` synchronisations per step and case.

`infer_multistep` replaces the whole of `test_multistep.infer` for an autoregressive model: the reference rolls out one
case at a time with B = 1 (`infer_case`, :102-132) and then synchronises three times per step and case; here the cases
run as one batched, graph-replayed rollout per chunk of at most `max_batch` cases, each followed by one metrics launch,
and the whole split makes one device->host copy.

`evaluate_auto` replaces `train_auto.evaluate` (reference src/train_auto.py:61-148), the single-step evaluation of the
dev split every `eval_interval` epochs and of the test split (with B = 1) after training: the reference builds every
batch on the host, runs one forward and synchronises 2 x (number of scores) times per batch; here chunks of up to
`max_batch` samples are gathered from device-resident frames, run as one forward each and reduced by one `fno_eval_sums`
launch per chunk, and the split makes one synchronisation.

`evaluate_rollout_auto` scores a split by rollout error, for choosing `train_auto` checkpoints of models trained
against rollout drift: every S-step window of the split rolls out from its start sample and each step is compared with
the true frame that many steps on.  Per chunk of windows one gather, one graph-replayed rollout and one
`fno_[grid_]window_metrics` launch that reads the targets straight from the device-resident frames; one
synchronisation for the split's chain check and one for the sums.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .data import (_check_chain, _check_grid, _check_split, _positive_int, as_device_frames, describe_split,
                   split_windows)

HW = 64 * 64


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


def _chunked_sums(host: np.ndarray, steps: int, n: int, max_batch: int) -> np.ndarray:
    """The (S, n, 3) sums of n items from the flat host copy of a device buffer that chunk [lo, hi) of at most
    max_batch items filled with its (S, hi - lo, 3) block at offset S*lo*3."""
    blocks = [host[steps * lo * 3:steps * min(n, lo + max_batch) * 3].reshape(steps, -1, 3)
              for lo in range(0, n, max_batch)]
    return np.concatenate(blocks, axis=1)


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
    preds = _lib.aligned(preds.float())
    label_u = _lib.aligned(label_u.to(preds.device).float())
    mask = _lib.aligned(mask.to(preds.device).float())
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
            label_u = _lib.aligned(fr[:, :, 0].transpose(0, 1))     # (S, B, H, W): frame s of each case
            mask = _lib.aligned(fr[:, :, 2].transpose(0, 1))
            _launch_metrics(preds, label_u, mask, sums[s * lo * 3:s * hi * 3])
    host = sums.double().cpu().numpy()   # the only synchronisation
    per_case = _per_case(_chunked_sums(host, s, n, max_batch), gh * gw)   # (S, n) each
    return [{k: float(np.mean(v[i])) for k, v in per_case.items()} for i in range(s)]


EVAL_SCORES = ("mse", "rmse", "mae", "nmse")   # what the reference's MseLoss.get_score_names can return


def _launch_eval_sums(preds: Tensor, label: Tensor, mask: Tensor, inputs: Tensor, sums: Tensor) -> None:
    """sums [B][6] (a contiguous float32 CUDA tensor or view) <- fno_eval_sums of the contiguous float32 CUDA tensors
    preds, label, inputs (B,2,H,W) and mask (B,1,H,W)."""
    b, _, gh, gw = preds.shape
    lib = _lib.load()
    with torch.cuda.device(preds.device):
        st = C.c_void_p(torch.cuda.current_stream(preds.device).cuda_stream)
        _lib.check(lib.fno_eval_sums(preds.data_ptr(), label.data_ptr(), mask.data_ptr(), inputs.data_ptr(),
                                     sums.data_ptr(), b, gh, gw, st), "fno_eval_sums")


def eval_scores(sums: np.ndarray, hw: int, batch_size: int, names: Sequence[str]) -> dict:
    """The `scores` of `train_auto.evaluate` (reference src/train_auto.py:75-147) from per-sample sums.

    sums: (N, 6) per-sample `fno_eval_sums` rows, hw = H*W.  The reference scores consecutive batches of `batch_size`
    samples (the last one may be short): per batch the model's loss on (preds, label * mask) over both channels and the
    input loss on (inputs[:, :1], label[:, :1]).  Each batch's sums are added in float64 in sample order; a batch whose
    labels are all zero gives the inf / nan of the reference's division.  Returns dict(mean={k, input_k: mean over
    batches}, all={k: [one score per batch]}), every value a Python float."""
    host = np.asarray(sums, dtype=np.float64)
    n = host.shape[0]
    n_full = n // batch_size
    tot = np.zeros((n_full, 6))
    if n_full:
        full = host[:n_full * batch_size].reshape(n_full, batch_size, 6)
        for j in range(batch_size):   # every full batch at once, its samples added in order
            tot += full[:, j]
    cnt = np.full(n_full, float(batch_size))
    if n % batch_size:                # the short last batch
        tot = np.concatenate([tot, np.cumsum(host[n_full * batch_size:], axis=0)[-1:]])
        cnt = np.append(cnt, float(n % batch_size))
    with np.errstate(divide="ignore", invalid="ignore"):
        per = {}
        for prefix, (e2, e1, l2), size in (("", (0, 1, 2), 2 * hw), ("input_", (3, 4, 5), hw)):
            mse = tot[:, e2] / (cnt * size)
            per[prefix] = dict(mse=mse, rmse=np.sqrt(mse), mae=tot[:, e1] / (cnt * size),
                               nmse=mse / (tot[:, l2] / (cnt * size)))
    scores = {k: per[""][k].tolist() for k in names}   # lists of Python floats
    mean = {}
    for k in names:
        mean[k] = float(np.mean(per[""][k]))
        mean[f"input_{k}"] = float(np.mean(per["input_"][k]))
    return dict(mean=mean, all=scores)


def evaluate_auto(model, data, batch_size: int = 2, max_batch: int = 256) -> dict:
    """What `train_auto.evaluate(model, data, output_dir, batch_size)` returns (reference src/train_auto.py:61-148),
    without its plots:  dict(preds=(2N, 1, H, W) float32 CPU tensor, scores=dict(mean=..., all=...)).

    data: the reference's dataset object (`.inputs`, `.labels` (N, 3, H, W), `.case_ids`, `.case_params`; uploaded once
    per call) or a `DeviceFrames` of it (built once, reused by every call).  The score names are
    `model.loss_fn.get_score_names()`, scored per reference batch of `batch_size` consecutive samples (see
    `eval_scores`).  `preds` are the masked predictions in sample order viewed as (-1, 1, H, W), as the reference's
    `preds.view(-1, 1, height, width)` gives them.  The model is put in eval mode and run under inference mode.

    Samples run in chunks of at most `max_batch`: per chunk one `DeviceFrames.batch` gather, one forward without label
    (the module's loss does not run), one `fno_eval_sums` launch into a device buffer for the whole split and one
    asynchronous copy of the predictions into a pinned host tensor; the split synchronises once, at the end.  Device
    memory beyond the frames and the (N, 6) sums is one chunk's worth.  Samples are computed independently, so the
    result does not depend on `max_batch`."""
    if batch_size < 1 or max_batch < 1:
        raise ValueError(f"batch_size and max_batch must be positive, got {batch_size} and {max_batch}")
    names = list(model.loss_fn.get_score_names())
    unknown = [k for k in names if k not in EVAL_SCORES]
    if unknown:
        raise ValueError(f"score names {unknown} are not among {EVAL_SCORES}")
    split = describe_split(data, "the split", nonempty=True)
    n, gh, gw = split.n, split.height, split.width
    _check_grid(gh, gw)
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise _lib.FnoNativeError("evaluate_auto has no CPU path: the model must be on a CUDA device")
    if split.device is not None and split.device != dev:
        raise ValueError(f"the split: the frames are on {split.device}, the model on {dev}")
    route = getattr(model, "_route", None)
    if route is not None:   # the drop-in Fno2d's own grid / storage-mode check, before any device work
        route(gh, gw)
    model.eval()
    preds_host = torch.empty(n, 2, gh, gw, dtype=torch.float32, pin_memory=True)   # a normal tensor, as torch.cat gives
    with torch.inference_mode(), torch.cuda.device(dev):
        frames = as_device_frames(data, dev)
        sums = torch.empty(n, 6, dtype=torch.float32, device=dev)
        for lo in range(0, n, max_batch):
            hi = min(n, lo + max_batch)
            batch = frames.batch(torch.arange(lo, hi).pin_memory())   # pinned: the index upload is asynchronous
            preds = model(inputs=batch["inputs"], case_params=batch["case_params"], mask=batch["mask"])["preds"]
            _launch_eval_sums(preds, batch["label"], batch["mask"], batch["inputs"], sums[lo:hi])
            preds_host[lo:hi].copy_(preds, non_blocking=True)
            del batch, preds
        host = sums.cpu().double().numpy()   # the only synchronisation
    return dict(preds=preds_host.view(-1, 1, gh, gw), scores=eval_scores(host, gh * gw, batch_size, names))


def rollout_scores(sums: np.ndarray, hw: int) -> dict:
    """The result of `evaluate_rollout_auto` from its window sums: sums (S, n, 3) float64, step k of window i in
    sums[k][i] (fno_[grid_]window_metrics' (sum (p-l)^2, sum l^2, sum |p-l|)), hw = H*W.  Per window and step the
    reference's get_metrics (`_per_case`: mse, nmse = mse / mean(l^2), mae); per step each the mean over the windows,
    added in float64 in window order; loss = the mean over the steps of nmse, added in step order.  A window whose
    label plane is all zero gives the inf / nan of the reference's division."""
    host = np.asarray(sums, dtype=np.float64)
    s, n = host.shape[:2]
    with np.errstate(divide="ignore", invalid="ignore"):
        per = _per_case(host, hw)   # (S, n) each
    steps = []
    for k in range(s):
        row = {}
        for name, v in per.items():
            tot = 0.0
            for x in v[k].tolist():   # window order
                tot += x
            row[name] = tot / n
        steps.append(row)
    loss = 0.0
    for row in steps:
        loss += row["nmse"]
    return dict(steps=steps, loss=loss / s, windows=int(n))


def _launch_window_metrics(frames, preds: Tensor, starts: Tensor, time_step_size: int, sums: Tensor) -> None:
    """sums [S][B][3] (a contiguous float32 CUDA tensor or view) <- fno_[grid_]window_metrics of the contiguous
    (S, B, 2, H, W) float32 rollout `preds` from the window starts `starts` ((B,) int64 on the device) of `frames`."""
    s, b, _, gh, gw = preds.shape
    lib = _lib.load()
    code = _lib.ACT_BF16 if frames.frame_dtype == torch.bfloat16 else _lib.ACT_F32
    args = (preds.data_ptr(), frames.frames_in.data_ptr(), frames.frames_out.data_ptr(), starts.data_ptr(), s, b,
            time_step_size, frames.n, code, sums.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream(preds.device).cuda_stream)
    if (gh, gw) == (64, 64):
        _lib.check(lib.fno_window_metrics(*args, st), "fno_window_metrics")
    else:
        _lib.check(lib.fno_grid_window_metrics(*args, gh, gw, st), "fno_grid_window_metrics")


def evaluate_rollout_auto(model, data, steps: int, time_step_size=None, max_batch: int = 256) -> dict:
    """The rollout error of `model` on a split: every window of `steps` = S samples inside one case rolls out S steps
    from its start sample, and step k (0-based) of the window that starts at sample j is compared with
    frames_out[j + k s] (s = `time_step_size`, by default the split's), the true frame k + 1 time steps on -- the
    targets `train_auto(rollout_steps=...)` trains against.  This is deliberately not test_multistep.infer's indexing,
    which compares prediction s with frame s of the case (`infer_multistep`).  Both sides are the u channel multiplied
    by the start sample's mask, the mask the rollout applies to its predictions.

    data: the reference's dataset object (uploaded once per call) or a `DeviceFrames` of it.  The windows are
    `rollout_windows(case_ids, S, s)`; the split must chain (frames_in[j + k s] == frames_out[j + (k-1) s] for every
    pair a window uses), which is checked on the device with one synchronisation.  model: the drop-in `Fno2d` on a
    CUDA device, in either storage mode; it is put in eval mode, and the gathers and metrics run under inference mode
    (the rollout's captured graph outlives the call, so it runs under no_grad, as `generate_many`).

    Windows run in chunks of at most `max_batch`: per chunk one `DeviceFrames.batch` gather of the start samples, one
    graph-replayed inference rollout (the kernels `generate_many` runs) whose contiguous (S, B, 2, H, W) output is read
    as it is, and one `fno_[grid_]window_metrics` launch into a device buffer for the whole split, which reads each
    target's u plane and the start mask from the frames: no label sequence is gathered.  The sums are copied to the
    host once, where `rollout_scores` reduces them in float64; with the chain check the call synchronises twice.
    Windows are computed independently, so the result does not depend on `max_batch`.

    Returns dict(steps=[{mse, nmse, mae} per step, each the mean over the windows], loss=the mean over the steps of
    nmse, windows=the window count).  Raises before any device work: TypeError for a model that is not the drop-in
    Fno2d; ValueError for a `steps`, `time_step_size` or `max_batch` that is not a positive int, no time step size at
    all, an empty or malformed split, a case-parameter count other than the model's, a grid or storage mode the model
    rejects, or a split without a single S-step window; FnoNativeError for a CPU model.  A split that does not chain
    raises ValueError naming the first bad sample."""
    from .fno2d import Fno2d
    steps = _positive_int("steps", steps)
    if time_step_size is not None:
        _positive_int("time_step_size", time_step_size)
    max_batch = _positive_int("max_batch", max_batch)
    if not isinstance(model, Fno2d):
        raise TypeError(f"evaluate_rollout_auto runs the drop-in cfdbench_b200.Fno2d, got {type(model).__name__}")
    split = _check_split(model, data, "the split")
    windows, tss = split_windows(split, steps, time_step_size, "the split", "steps")
    model._require_cuda()
    with torch.inference_mode(), torch.cuda.device(model.device):
        frames = as_device_frames(data, model.device)
        _check_chain(frames, windows, steps, tss, what="the split")
    return _evaluate_rollout(model, frames, windows, steps, tss, max_batch)


def _evaluate_rollout(model, frames, windows: np.ndarray, steps: int, time_step_size: int, max_batch: int = 256) -> dict:
    """evaluate_rollout_auto on checked arguments: `frames` a DeviceFrames on the model's device, `windows` its
    S-step window starts, the chain already checked."""
    model.eval()
    with torch.inference_mode(), torch.cuda.device(model.device):
        sums = _window_sums(model, frames, windows, steps, time_step_size, max_batch)
    return rollout_scores(sums, frames.height * frames.width)


def _window_sums(model, frames, windows: np.ndarray, steps: int, time_step_size: int, max_batch: int) -> np.ndarray:
    """The (S, n, 3) float64 fno_[grid_]window_metrics sums of the windows starting at `windows` (checked: inside one
    case each, the split chaining), in window order: per chunk of at most max_batch windows one gather, one rollout and
    one metrics launch; one synchronisation.  Runs in the caller's inference mode and device context."""
    dev, n = model.device, int(windows.size)
    sums = torch.empty(steps * n * 3, dtype=torch.float32, device=dev)   # chunk [lo, hi)'s (S, B, 3) at S*lo*3
    for lo in range(0, n, max_batch):
        hi = min(n, lo + max_batch)
        starts = torch.from_numpy(windows[lo:hi]).pin_memory()   # pinned: the index uploads are asynchronous
        b0 = frames.batch(starts)
        with torch.inference_mode(False), torch.no_grad():   # the captured rollout's static buffers outlive the call
            x, cp, mk = model._prep_inputs(b0["inputs"], b0["case_params"], b0["mask"])
            preds = model._rollout_device(x, cp, mk, steps)     # (S, B, 2, H, W), contiguous
        _launch_window_metrics(frames, preds, starts.to(dev, non_blocking=True), time_step_size,
                               sums[steps * lo * 3:steps * hi * 3])
        del b0, preds
    return _chunked_sums(sums.cpu().double().numpy(), steps, n, max_batch)   # the one synchronisation
