"""Device-resident input pipeline (SURVEY.md 8f.2).

The reference holds every (input, label) frame pair of a split in two host tensors `dataset.inputs` /
`dataset.labels` of shape (N, 3, h, w) (u, v, mask), a per-sample `dataset.case_ids` and a list of per-case parameter
dicts `dataset.case_params` (src/dataset/cavity.py:283-331, cylinder.py likewise); `DataLoader` + `collate_fn`
(src/train_auto.py:33-58, 208-210) then builds each batch on the host and copies it to the GPU.  `DeviceFrames`
uploads the split once (fp32, or bf16 to halve its footprint) and produces the same batch dict with one kernel launch
(`fno_gather_batch`); the on-disk format and the dataset classes are untouched -- it takes the dataset object as is.
Frames are 64x64 (cavity, cylinder) or any H x W with 24 <= H, W <= 128 (`fno_grid_gather_batch`; the tube and dam
datasets hold (N, 3, 66, 65) frames, reference src/dataset/tube.py:228-281, dam.py:275-313).

    frames = DeviceFrames(train_data, device="cuda")
    for batch in frames.loader(batch_size=32, shuffle=True, generator=g):   # same index order as the DataLoader
        out = model(**batch)
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, Iterator, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

EXCLUDED_KEYS = ("rotated", "dx", "dy")  # collate_fn, reference src/train_auto.py:45-47


def case_table(case_params: Sequence[dict]) -> np.ndarray:
    """(n_cases, p) float32 table with collate_fn's key order: the keys of the first dict minus EXCLUDED_KEYS."""
    keys = [k for k in case_params[0].keys() if k not in EXCLUDED_KEYS]
    return np.asarray([[cp[k] for k in keys] for cp in case_params], dtype=np.float32).reshape(len(case_params), len(keys))


def _positive_int(name: str, v) -> int:
    """`v` as an int; ValueError unless it is a positive int (a bool is not)."""
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
        raise ValueError(f"{name} must be a positive int, got {v!r}")
    return int(v)


def _check_grid(gh: int, gw: int) -> None:
    """ValueError for a grid outside the grid-generic kernels' range (64x64 lies inside it)."""
    from . import _lib
    if not (_lib.GRID_MIN <= gh <= _lib.GRID_MAX and _lib.GRID_MIN <= gw <= _lib.GRID_MAX):
        raise ValueError(f"grid {gh}x{gw} is outside the supported range {_lib.GRID_MIN}..{_lib.GRID_MAX} in H and W")


class DeviceFrames:
    def __init__(self, dataset, device="cuda", frame_dtype: torch.dtype = torch.float32):
        if frame_dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("frame_dtype must be float32 or bfloat16")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("DeviceFrames keeps the split in GPU memory: pass a CUDA device")
        split = describe_split(dataset, "dataset")
        _check_grid(split.height, split.width)
        self.n, self.height, self.width, self.n_case_params = split.n, split.height, split.width, split.n_case_params
        self.device, self.frame_dtype = dev, frame_dtype
        from . import _lib
        self.frames_in = _lib.aligned(dataset.inputs.to(device=dev, dtype=frame_dtype))   # the gathers' vector reads
        self.frames_out = _lib.aligned(dataset.labels.to(device=dev, dtype=frame_dtype))
        self.case_table = torch.from_numpy(case_table(dataset.case_params)).to(dev)
        self.case_ids = torch.as_tensor(split.case_ids, dtype=torch.int32, device=dev)
        self._case_ids_host = split.case_ids   # for the window checks, without a device read
        # the dataset's label offset (labels = frames[s:], inputs = frames[:-s] per case), None when it has none
        self.time_step_size = split.time_step_size

    def __len__(self) -> int:
        return self.n

    def batch(self, idx, noise_std: float = 0.0, noise_seed: int = 0, noise_step: int = 0) -> Dict[str, Tensor]:
        """The dict collate_fn returns for samples `idx` (reference src/train_auto.py:53-58), all on the device.

        noise_std > 0 then adds seeded Gaussian noise to the input frames where the mask is non-zero, one more launch
        (`fno_add_input_noise`): inputs += noise_std * z * mask, z a pure function of (noise_seed, noise_step, the sample
        index, the element), so the same sample gets the same noise in any batch.  Labels, mask and case parameters are
        not perturbed; noise_std = 0 launches nothing extra.  `train_auto(input_noise_std=...)` passes Adam's 1-based
        step as noise_step.  Raises ValueError for a negative or non-finite noise_std, a noise_seed outside [0, 2^64)
        or a noise_step outside [0, 2^63)."""
        from . import _lib
        noise_std = check_noise_args(noise_std, noise_seed, noise_step)
        _lib.load()   # a missing library raises before any device work
        idx = torch.as_tensor(idx, dtype=torch.int64)
        if idx.dim() != 1 or idx.numel() == 0:
            raise ValueError("idx must be a non-empty 1-D index list")
        if int(idx.min()) < 0 or int(idx.max()) >= self.n:
            raise IndexError("sample index out of range")
        idx = idx.to(self.device, non_blocking=True)
        b, p, dev, gh, gw = idx.numel(), self.n_case_params, self.device, self.height, self.width
        out = dict(inputs=torch.empty(b, 2, gh, gw, device=dev), label=torch.empty(b, 2, gh, gw, device=dev),
                   mask=torch.empty(b, 1, gh, gw, device=dev), case_params=torch.empty(b, p, device=dev))
        with torch.cuda.device(dev):
            st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _gather(self, idx, b, out["inputs"], out["label"], out["mask"], out["case_params"], st)
            if noise_std > 0:
                self._add_noise(out, idx, noise_std, noise_seed, noise_step, st)
        idx.record_stream(torch.cuda.current_stream(dev))
        return out

    def _add_noise(self, out: Dict[str, Tensor], idx: Tensor, std: float, seed: int, step: int, st) -> None:
        from . import _lib
        step_dev = torch.full((1,), int(step), dtype=torch.int64, device=self.device)   # a fill kernel, no copy
        _lib.check(_lib.load().fno_add_input_noise(out["inputs"].data_ptr(), out["mask"].data_ptr(), idx.data_ptr(),
                                                   idx.numel(), self.height, self.width, std, int(seed),
                                                   step_dev.data_ptr(), None, st), "fno_add_input_noise")

    def rollout_batch(self, idx, steps: int, time_step_size=None, noise_std: float = 0.0, noise_seed: int = 0,
                      noise_step: int = 0) -> Dict[str, Tensor]:
        """`batch(idx)` for the windows that start at samples `idx`, plus "labels" (steps, B, 2, H, W): step k's target
        labels[idx + k s] * mask, masked with the start sample's mask as `Fno2d.rollout` masks its predictions
        (s = time_step_size, by default the dataset's).  One launch (fno_[grid_]gather_window).

            b = frames.rollout_batch(idx, K)
            preds = model.rollout(b["inputs"], b["case_params"], b["mask"], K)
            loss = sum(model.loss_fn(preds=preds[k], labels=b["labels"][k])["nmse"] for k in range(K)) / K

        noise_std, noise_seed and noise_step perturb the start samples' input frames as in `batch`; the targets are
        not perturbed.

        Raises ValueError for a non-positive steps / time_step_size, no time_step_size at all, a window that crosses
        a case boundary or bad noise arguments (as `batch`); IndexError for a window that runs past the split."""
        from . import _lib
        noise_std = check_noise_args(noise_std, noise_seed, noise_step)
        _lib.load()   # a missing library raises before any device work
        s = self.time_step_size if time_step_size is None else time_step_size
        steps = _positive_int("steps", steps)
        if s is None:
            raise ValueError("time_step_size is needed: the dataset has none, pass it")
        s = _positive_int("time_step_size", s)
        idx = torch.as_tensor(idx, dtype=torch.int64)
        if idx.dim() != 1 or idx.numel() == 0:
            raise ValueError("idx must be a non-empty 1-D index list")
        starts = idx.cpu().numpy()
        ends = starts + (steps - 1) * s
        if int(starts.min()) < 0 or int(ends.max()) >= self.n:
            raise IndexError("sample index out of range, or a window runs past the split")
        cross = np.flatnonzero(self._case_ids_host[starts] != self._case_ids_host[ends])
        if cross.size:
            raise ValueError(f"the {steps}-step window that starts at sample {int(starts[cross[0]])} crosses a case boundary")
        idx = idx.to(self.device, non_blocking=True)
        b, p, dev, gh, gw = idx.numel(), self.n_case_params, self.device, self.height, self.width
        out = dict(inputs=torch.empty(b, 2, gh, gw, device=dev), label=torch.empty(b, 2, gh, gw, device=dev),
                   mask=torch.empty(b, 1, gh, gw, device=dev), case_params=torch.empty(b, p, device=dev),
                   labels=torch.empty(steps, b, 2, gh, gw, device=dev))
        with torch.cuda.device(dev):
            st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _gather(self, idx, b, out["inputs"], out["label"], out["mask"], out["case_params"], st,
                    window=(steps, s, out["labels"]))
            if noise_std > 0:
                self._add_noise(out, idx, noise_std, noise_seed, noise_step, st)
        idx.record_stream(torch.cuda.current_stream(dev))
        return out

    def batches(self, index_batches: Iterable[Sequence[int]]) -> Iterator[Dict[str, Tensor]]:
        for ib in index_batches:
            yield self.batch(ib)

    def loader(self, batch_size: int, shuffle: bool = False, generator=None, drop_last: bool = False):
        """Batches in exactly the order `DataLoader(dataset, batch_size, shuffle, generator=generator)` visits them:
        the index stream comes from the same torch samplers the DataLoader builds (`index_batches`)."""
        return self.batches(index_batches(self.n, batch_size, shuffle, generator, drop_last))


def _gather(frames: DeviceFrames, idx: Tensor, b: int, inputs: Tensor, label: Optional[Tensor], mask: Tensor,
            case_params: Tensor, st, window: tuple = ()) -> None:
    """One launch that gathers samples idx[:b] of `frames` into the batch buffers, chosen by the frames' shape:
    fno_gather_batch on 64x64 frames, fno_grid_gather_batch on any other grid.  window = (steps, time_step_size, labels)
    gathers the windows that start there (fno_[grid_]gather_window), each step's masked target into `labels`; `label`
    may then be None."""
    from . import _lib
    args = (frames.frames_in.data_ptr(), frames.frames_out.data_ptr(), frames.case_table.data_ptr(),
            frames.case_ids.data_ptr(), idx.data_ptr(), b, frames.n_case_params,
            _lib.ACT_BF16 if frames.frame_dtype == torch.bfloat16 else _lib.ACT_F32, inputs.data_ptr(),
            None if label is None else label.data_ptr(), mask.data_ptr(), case_params.data_ptr())
    name = "gather_batch"
    if window:
        steps, s, labels = window
        args += (steps, s, frames.n, labels.data_ptr())
        name = "gather_window"
    lib, gh, gw = _lib.load(), frames.height, frames.width
    if (gh, gw) == (64, 64):
        name = "fno_" + name
        _lib.check(getattr(lib, name)(*args, st), name)
    else:
        name = "fno_grid_" + name
        _lib.check(getattr(lib, name)(*args, gh, gw, st), name)


class SplitInfo(NamedTuple):
    """What `describe_split` reads of a split."""
    n: int
    height: int
    width: int
    n_case_params: int
    frame_dtype: torch.dtype         # the frames' storage: float32 for a dataset object, which is uploaded so
    case_ids: np.ndarray             # (n,), on the host
    time_step_size: Optional[int]    # the split's label offset, None when it has none
    device: Optional[torch.device]   # the frames' device (with its index), None for a dataset object


def describe_split(data, what: str, nonempty: bool = False) -> SplitInfo:
    """The facts of a split: a DeviceFrames, or the reference's dataset object (`.inputs` / `.labels` (N, 3, H, W)
    tensors, `.case_ids`, `.case_params`, optionally `.time_step_size`).  No device work.  Raises ValueError, naming the
    split `what`, for a dataset whose frames are malformed or whose case_ids do not have one entry per sample, and with
    nonempty=True for a split without samples."""
    if isinstance(data, DeviceFrames):
        n = data.n
    else:
        ins, labs = getattr(data, "inputs", None), getattr(data, "labels", None)
        if not isinstance(ins, Tensor) or not isinstance(labs, Tensor) or ins.dim() != 4 or ins.shape[1] != 3 \
                or labs.shape != ins.shape:
            raise ValueError(f"{what} must be a dataset with (N, 3, H, W) .inputs / .labels tensors, got "
                             f"{getattr(ins, 'shape', None)} / {getattr(labs, 'shape', None)}")
        n = int(ins.shape[0])
    if nonempty and n == 0:   # before the case table: an empty dataset may have no case parameters
        raise ValueError(f"{what} is empty")
    tss = getattr(data, "time_step_size", None)
    if isinstance(data, DeviceFrames):
        frames_in = getattr(data, "frames_in", None)   # None on a DeviceFrames made without __init__
        return SplitInfo(n, data.height, data.width, data.n_case_params, data.frame_dtype, data._case_ids_host, tss,
                         None if frames_in is None else frames_in.device)
    ids = np.asarray(data.case_ids).reshape(-1)
    if ids.size != n:
        raise ValueError(f"{what} must have one case_ids entry per sample")
    return SplitInfo(n, int(ins.shape[2]), int(ins.shape[3]), case_table(data.case_params).shape[1], torch.float32, ids,
                     tss, None)


def _check_split(model, data, what: str) -> SplitInfo:
    """`describe_split(data, what, nonempty=True)`, refusing also a split the drop-in Fno2d `model` cannot train or
    evaluate on: frames on another device than the model, a case-parameter count other than the model's, or a grid /
    storage mode the model rejects.  No device work."""
    split = describe_split(data, what, nonempty=True)
    if split.device is not None and split.device != model.device:
        raise ValueError(f"{what}: the frames are on {split.device}, the model on {model.device}")
    if split.n_case_params != model.n_case_params:
        raise ValueError(f"{what} has {split.n_case_params} case parameters per sample, the model takes n_case_params="
                         f"{model.n_case_params}")
    model._route(split.height, split.width)   # the model's own grid / storage-mode checks
    return split


def as_device_frames(data, device) -> DeviceFrames:
    """`data` if it is a DeviceFrames, else a DeviceFrames of it on `device` (float32 frames)."""
    return data if isinstance(data, DeviceFrames) else DeviceFrames(data, device=device)


def check_noise_args(noise_std, noise_seed, noise_step=0, std_name: str = "noise_std") -> float:
    """Refuse training-noise arguments the noise kernel cannot take: a noise_std that is not a real >= 0 and finite in
    float32, a
    noise_seed that is not an int in [0, 2^64), a noise_step that is not an int in [0, 2^63).  Returns noise_std as a
    float."""
    if isinstance(noise_std, bool) or not isinstance(noise_std, (int, float, np.integer, np.floating)) \
            or not np.isfinite(noise_std) or noise_std < 0 or noise_std > float(np.finfo(np.float32).max):
        raise ValueError(f"{std_name} must be a real number >= 0, finite in float32, got {noise_std!r}")
    for name, v, hi in (("noise_seed", noise_seed, 2 ** 64), ("noise_step", noise_step, 2 ** 63)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= int(v) < hi:
            raise ValueError(f"{name} must be an int in [0, 2^{hi.bit_length() - 1}), got {v!r}")
    return float(noise_std)


class RolloutNoise(NamedTuple):
    """The per-step input noise of `Fno2d.rollout(noise=...)`: Gaussian noise of standard deviation `std` from the
    counter-based RNG of `add_input_noise`, keyed by `seed` and counted by `step` (train_auto passes Adam's 1-based
    step), `ids` ((B,) int64 on the model's device: each sample's dataset index, so the noise does not depend on the
    batch slot) and the noise stream; rollout step s draws from stream k0 + s."""
    std: float
    seed: int
    step: int
    ids: Tensor
    k0: int = 0


def check_rollout_noise(noise, batch: int, steps) -> Optional[RolloutNoise]:
    """Refuse a `Fno2d.rollout` noise record the native drivers cannot take: not a RolloutNoise, noise arguments
    `check_noise_args` refuses, ids that are not a (batch,) int64 tensor, or a k0 that is not an int >= 0 with
    k0 + steps <= 2^16 (the streams).  Returns None for no noise (None, or std 0: the path without noise), else the
    record with std as a float and the ints as Python ints."""
    if noise is None:
        return None
    if not isinstance(noise, RolloutNoise):
        raise ValueError(f"noise must be a RolloutNoise or None, got {type(noise).__name__}")
    std = check_noise_args(noise.std, noise.seed, noise.step)
    ids, k0 = noise.ids, noise.k0
    if not isinstance(ids, Tensor) or ids.dtype != torch.int64 or tuple(ids.shape) != (batch,):
        raise ValueError(f"noise.ids must be a ({batch},) int64 tensor, got "
                         f"{getattr(ids, 'dtype', type(ids).__name__)} {tuple(getattr(ids, 'shape', ()))}")
    n_steps = steps if isinstance(steps, int) and not isinstance(steps, bool) else 1
    if isinstance(k0, bool) or not isinstance(k0, (int, np.integer)) or k0 < 0 or int(k0) + n_steps > 2 ** 16:
        raise ValueError(f"noise.k0 must be an int >= 0 with k0 + steps <= 2^16, got {k0!r} with steps={steps!r}")
    if std == 0:
        return None
    return RolloutNoise(std, int(noise.seed), int(noise.step), ids.contiguous(), int(k0))


class _NoiseFn(torch.autograd.Function):
    """frames + noise with the identity as its gradient w.r.t. the frames (the noise does not depend on them)."""

    @staticmethod
    def forward(ctx, frames: Tensor, noise_args: tuple) -> Tensor:
        return _noise_out_of_place(frames, *noise_args)

    @staticmethod
    def backward(ctx, grad: Tensor):
        return grad, None


def _noise_out_of_place(frames: Tensor, mask: Tensor, ids: Tensor, std: float, seed: int, step: int,
                        stream: int) -> Tensor:
    from . import _lib
    out = torch.empty_like(frames)
    b, _, gh, gw = frames.shape
    with torch.cuda.device(frames.device):
        step_dev = torch.full((1,), step, dtype=torch.int64, device=frames.device)   # a fill kernel, no copy
        st = C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)
        _lib.check(_lib.load().fno_add_input_noise_stream(frames.data_ptr(), out.data_ptr(), mask.data_ptr(), ids.data_ptr(),
                                                          b, gh, gw, std, seed, step_dev.data_ptr(), None, stream, st),
                   "fno_add_input_noise_stream")
    return out


def add_input_noise(frames: Tensor, mask: Tensor, ids: Tensor, std: float, seed: int, step: int,
                    stream: int = 0) -> Tensor:
    """A new tensor: `frames` ((B, 2, H, W) float32 on a CUDA device) plus seeded Gaussian noise where `mask` ((B, 1, H,
    W) or (B, H, W)) is non-zero, `frames` elsewhere.  The noise is that of `DeviceFrames.batch(noise_std=std,
    noise_seed=seed, noise_step=step)` for the samples with dataset indices `ids` ((B,) int64), drawn from noise stream
    `stream` (0 <= stream < 2^16): stream 0 is exactly the noise `batch` adds, and `Fno2d.rollout(noise=RolloutNoise(std,
    seed, step, ids, k0))` feeds its step s a frame perturbed with stream k0 + s.  One launch
    (`fno_add_input_noise_stream`).  Differentiable w.r.t. `frames`, with the identity as gradient.  Raises ValueError
    for bad noise arguments (as `DeviceFrames.batch`), a stream outside 0 .. 2^16 - 1 or mismatched shapes."""
    std = check_noise_args(std, seed, step, std_name="std")
    if isinstance(stream, bool) or not isinstance(stream, (int, np.integer)) or not 0 <= stream < 2 ** 16:
        raise ValueError(f"stream must be an int in [0, 2^16), got {stream!r}")
    if not isinstance(frames, Tensor) or frames.dim() != 4 or frames.shape[1] != 2 or frames.dtype != torch.float32:
        raise ValueError(f"frames must be a (B, 2, H, W) float32 tensor, got {getattr(frames, 'shape', None)}")
    b, _, gh, gw = frames.shape
    if mask.shape not in ((b, 1, gh, gw), (b, gh, gw)):
        raise ValueError(f"mask must be ({b}, 1, {gh}, {gw}) or ({b}, {gh}, {gw}), got {tuple(mask.shape)}")
    if not isinstance(ids, Tensor) or ids.dtype != torch.int64 or tuple(ids.shape) != (b,):
        raise ValueError(f"ids must be a ({b},) int64 tensor")
    if frames.device.type != "cuda" or mask.device != frames.device or ids.device != frames.device:
        raise ValueError("frames, mask and ids must be on the same CUDA device")
    args = (mask.to(torch.float32).contiguous(), ids.contiguous(), std, int(seed), int(step), int(stream))
    if frames.requires_grad and torch.is_grad_enabled():
        return _NoiseFn.apply(frames.contiguous(), args)
    return _noise_out_of_place(frames.detach().contiguous(), *args)


class TeacherForcing(NamedTuple):
    """The teacher forcing of `Fno2d.rollout(teacher=...)` (scheduled sampling): `frames` ((steps - 1, B, 2, H, W)
    float32 on the model's device) are the true frames and `flags` ((steps - 1, B) bool or uint8, same device) choose
    them: rollout step s >= 1 of sample b is fed frames[s - 1][b] where flags[s - 1][b] is set, else the prediction of
    step s - 1.  With `rollout_batch`'s window, frames = b["labels"][:steps - 1] (the masked targets) and flags from
    `teacher_forcing_flags`."""
    frames: Tensor
    flags: Tensor


def check_teacher_forcing(teacher, batch: int, steps, gh: int, gw: int) -> Optional[TeacherForcing]:
    """Refuse a `Fno2d.rollout` teacher record the native drivers cannot take: not a TeacherForcing, steps < 2, frames
    that are not a (steps - 1, batch, 2, gh, gw) float32 tensor or that require grad (the true frames are data), flags
    that are not a (steps - 1, batch) bool or uint8 tensor, or the two on different devices.  Returns None for None,
    else the record with contiguous frames and uint8 flags."""
    if teacher is None:
        return None
    if not isinstance(teacher, TeacherForcing):
        raise ValueError(f"teacher must be a TeacherForcing or None, got {type(teacher).__name__}")
    if isinstance(steps, bool) or not isinstance(steps, int) or steps < 2:
        raise ValueError(f"teacher forcing needs steps >= 2 (step 0 is always fed the start frame), got steps={steps!r}")
    frames, flags = teacher.frames, teacher.flags
    shape = (steps - 1, batch, 2, gh, gw)
    if not isinstance(frames, Tensor) or frames.dtype != torch.float32 or tuple(frames.shape) != shape:
        raise ValueError(f"teacher.frames must be a {shape} float32 tensor, got "
                         f"{getattr(frames, 'dtype', type(frames).__name__)} {tuple(getattr(frames, 'shape', ()))}")
    if frames.requires_grad:
        raise ValueError("teacher.frames requires grad: the true frames are data, and no gradient flows into them")
    if not isinstance(flags, Tensor) or flags.dtype not in (torch.bool, torch.uint8) or \
            tuple(flags.shape) != (steps - 1, batch):
        raise ValueError(f"teacher.flags must be a ({steps - 1}, {batch}) bool or uint8 tensor, got "
                         f"{getattr(flags, 'dtype', type(flags).__name__)} {tuple(getattr(flags, 'shape', ()))}")
    if flags.device != frames.device:
        raise ValueError(f"teacher.frames is on {frames.device}, teacher.flags on {flags.device}")
    return TeacherForcing(frames.contiguous(), flags.to(torch.uint8).contiguous())


def check_teacher_prob(prob, name: str = "prob") -> float:
    """A teacher-forcing probability: a real number in [0, 1].  Returns it as a float."""
    if isinstance(prob, bool) or not isinstance(prob, (int, float, np.integer, np.floating)) \
            or not np.isfinite(prob) or not 0 <= prob <= 1:
        raise ValueError(f"{name} must be a real number in [0, 1], got {prob!r}")
    return float(prob)


def teacher_forcing_flags(ids: Tensor, steps: int, prob: float, seed: int, step: int) -> Tensor:
    """The (steps - 1, B) uint8 teacher-forcing flags of windows that start at dataset indices `ids` ((B,) int64 on a
    CUDA device): flags[s - 1][b] = 1 with probability `prob`, drawn from the counter-based RNG of `add_input_noise`
    keyed by `seed` and counted by `step` (train_auto passes Adam's 1-based step), a pure function of (seed, step,
    ids[b], s) whatever the batch slot.  prob = 0 sets no flag, prob = 1 every flag.  One launch
    (`fno_teacher_flags`); train_auto(teacher_forcing=p, teacher_seed=seed) draws exactly these.  Raises ValueError for
    steps < 2, a prob outside [0, 1], a seed outside [0, 2^64), a step outside [0, 2^63) or malformed ids."""
    from . import _lib
    if isinstance(steps, bool) or not isinstance(steps, (int, np.integer)) or not 2 <= steps <= 2 ** 16:
        raise ValueError(f"steps must be an int in [2, 2^16], got {steps!r}")
    prob = check_teacher_prob(prob)
    for name, v, hi in (("seed", seed, 2 ** 64), ("step", step, 2 ** 63)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= int(v) < hi:
            raise ValueError(f"{name} must be an int in [0, 2^{hi.bit_length() - 1}), got {v!r}")
    if not isinstance(ids, Tensor) or ids.dtype != torch.int64 or ids.dim() != 1 or ids.numel() < 1 \
            or ids.device.type != "cuda":
        raise ValueError("ids must be a non-empty (B,) int64 tensor on a CUDA device")
    ids = ids.contiguous()
    b = ids.numel()
    out = torch.empty(int(steps) - 1, b, dtype=torch.uint8, device=ids.device)
    with torch.cuda.device(ids.device):
        step_dev = torch.full((1,), int(step), dtype=torch.int64, device=ids.device)   # fill kernels, no copies
        prob_dev = torch.full((1,), prob, dtype=torch.float32, device=ids.device)
        st = C.c_void_p(torch.cuda.current_stream(ids.device).cuda_stream)
        _lib.check(_lib.load().fno_teacher_flags(ids.data_ptr(), b, int(steps), prob_dev.data_ptr(), int(seed),
                                                 step_dev.data_ptr(), None, out.data_ptr(), st), "fno_teacher_flags")
    return out


def index_batches(n: int, batch_size: int, shuffle: bool = False, generator=None,
                  drop_last: bool = False) -> Iterator[List[int]]:
    """The index batches one iteration of `DataLoader(dataset_of_len_n, batch_size, shuffle, generator=generator,
    drop_last=drop_last)` yields, drawing from the RNG (`generator`, or the global one for None) exactly what that
    iteration draws.  Lazy, like the DataLoader iterator: nothing is drawn before the first batch is requested."""
    from torch.utils.data import BatchSampler, RandomSampler, SequentialSampler
    base: List[int] = list(range(n))
    sampler = RandomSampler(base, generator=generator) if shuffle else SequentialSampler(base)

    def gen():
        # a DataLoader iterator draws its worker base seed from the generator before the sampler draws the
        # permutation (torch/utils/data/dataloader.py, _BaseDataLoaderIter.__init__); do the same so that the RNG
        # stream, and with it the visiting order, is identical
        torch.empty((), dtype=torch.int64).random_(generator=generator)
        yield from BatchSampler(sampler, batch_size, drop_last)
    return gen()


def rollout_windows(case_ids, steps: int, time_step_size: int) -> np.ndarray:
    """The valid starts (int64, ascending) of `steps`-step windows over a split whose samples are laid out as the
    reference's datasets lay them out: a case's samples are contiguous, with inputs = frames[:-s] and labels = frames[s:]
    (s = time_step_size, src/dataset/cavity.py:271,295-331), so the k-th target of the window that starts at sample j is
    labels[j + k s].  A start j is valid when j + (steps - 1) s < N and case_ids[j + (steps - 1) s] == case_ids[j]: no
    window crosses a case.  steps = 1 gives arange(N)."""
    steps, time_step_size = _positive_int("steps", steps), _positive_int("time_step_size", time_step_size)
    span = (steps - 1) * time_step_size
    cid = np.asarray(case_ids).reshape(-1)
    if cid.size <= span:
        return np.zeros(0, dtype=np.int64)
    j = np.arange(cid.size - span, dtype=np.int64)
    return j[cid[j + span] == cid[j]]


def split_windows(split: SplitInfo, steps: int, time_step_size, what: str, steps_name: str) -> Tuple[np.ndarray, int]:
    """(windows, s): the `rollout_windows` of `split` for `steps`-step rollouts and their time step size s, the
    `time_step_size` argument unless it is None, else the split's.  ValueError, naming the split `what` and the steps
    argument `steps_name`, for no time step size at all, one that is not a positive int, or no single window."""
    s = split.time_step_size if time_step_size is None else time_step_size
    if s is None:
        raise ValueError(f"{steps_name}={steps} needs a time_step_size: {what} has none, pass it")
    windows = rollout_windows(split.case_ids, steps, s)
    if windows.size == 0:
        raise ValueError(f"{what} has no {steps}-step window with time_step_size={s} inside one case")
    return windows, int(s)


def _check_chain(frames: DeviceFrames, starts: np.ndarray, steps: int, time_step_size: int,
                 what: str = "train_data") -> None:
    """Refuse a split whose frames do not chain where the windows starting at `starts` need them to: step k of the
    window at j is fed the prediction of step k-1 where the data has frames_in[j + k s], and trained against
    frames_out[j + (k-1) s], so the two must be the same frame (bit for bit, mask channel included).  Compared on the
    device in chunks; one synchronisation for the whole check.  The error names the split (`what`) and the
    first bad sample."""
    s, dev, n = time_step_size, frames.device, frames.n
    rows = np.unique((starts[:, None] + s * np.arange(steps - 1, dtype=np.int64)[None, :]).ravel())
    host = torch.from_numpy(rows).pin_memory()
    rows_dev = host.to(dev, non_blocking=True)
    bits = torch.int32 if frames.frame_dtype == torch.float32 else torch.int16
    first = torch.full((), n, dtype=torch.int64, device=dev)
    chunk = 512
    for c0 in range(0, rows.size, chunk):
        i = rows_dev[c0:c0 + chunk]
        a = frames.frames_in.index_select(0, i + s).view(bits)
        b = frames.frames_out.index_select(0, i).view(bits)
        bad = (a != b).flatten(1).any(1)
        first = torch.minimum(first, torch.where(bad, i, first).min())
    bad_row = int(first)   # the check's one synchronisation
    if bad_row < n:
        raise ValueError(f"{what} does not chain with time_step_size={s}: sample {bad_row + s}'s input frame is not "
                         f"sample {bad_row}'s label frame, which a {steps}-step rollout window feeds it")
