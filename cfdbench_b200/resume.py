"""The training state `train_auto(..., resumable=True)` keeps beside its checkpoints, so that relaunching the same call
continues an interrupted run bit for bit instead of starting a different one.

One file, `output_dir / "training_state.pt"`, overwritten atomically at the end of every evaluation epoch and after the
last epoch.  It loads with `torch.load(..., weights_only=True)`: tensors, numbers, strings, lists, tuples and dicts only.

    version       STATE_VERSION
    epoch         the last completed epoch (0-based)
    global_step   Adam's step count after that epoch
    model         the trained weights' state_dict (never the EMA copy)
    optimizer     FusedAdam.state_dict(): step, exp_avg, exp_avg_sq [, ema] per trainable parameter
    scheduler     StepLR.state_dict()
    rng           "generator" or "global": which RNG the visiting order draws from
    rng_state     that RNG's state after the epoch's draws (generator.get_state() / torch.get_rng_state())
    train_losses  every step's loss so far
    grad_norms    every step's pre-clip gradient norm so far (with max_grad_norm only)
    config        run_config(...): every setting the trajectory or the checkpoint scores depend on, compared on resume
                  (random_unroll and unroll_seed only in the record of a random_unroll=True run)
"""
from __future__ import annotations

import hashlib
import os
import tempfile
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from .data import DeviceFrames, describe_split  # noqa: F401  (DeviceFrames is re-exported)

STATE_NAME = "training_state.pt"
STATE_VERSION = 1


def model_config(model) -> dict:
    """The Fno2d settings that change what a training step computes: shapes, storage mode, the kernel choices that
    change the arithmetic and which parameters are trained."""
    return dict(in_chan=model.in_chan, out_chan=model.out_chan, n_case_params=model.n_case_params,
                num_layers=model.num_layers, hidden_dim=model.hidden_dim, modes1=model.modes1, modes2=model.modes2,
                act_dtype=model.act_dtype, fused_block=bool(model.fused_block),
                generic_grid_at_64=bool(model.generic_grid_at_64),
                requires_grad=[bool(p.requires_grad) for p in model.parameters()])


def split_fingerprint(data) -> dict:
    """Sample count, grid, case-parameter count, frame storage dtype and a SHA-256 of the case_ids sequence of a split
    (`describe_split`: a DeviceFrames or the reference's dataset object, which train_auto uploads in float32).  The
    frames themselves are not hashed."""
    split = describe_split(data, "data")
    ids = np.ascontiguousarray(split.case_ids, dtype=np.int64)
    return dict(n=int(split.n), height=int(split.height), width=int(split.width), n_case_params=int(split.n_case_params),
                frame_dtype=str(split.frame_dtype).replace("torch.", ""),
                case_ids_sha256=hashlib.sha256(ids.tobytes()).hexdigest())


def run_config(model, train_data, dev_data, **args) -> dict:
    """The state's config record: model_config as "model.<field>", the run's arguments `args` (plain Python values) as
    given, and each split's fingerprint as "train_data.<field>" / "dev_data.<field>"."""
    cfg = {f"model.{k}": v for k, v in model_config(model).items()}
    cfg.update(args)
    for what, data in (("train_data", train_data), ("dev_data", dev_data)):
        cfg.update({f"{what}.{k}": v for k, v in split_fingerprint(data).items()})
    return cfg


def check_config(saved: dict, config: dict, path) -> None:
    """ValueError naming every field whose saved value differs from this call's (or is missing from either)."""
    def show(d, k):
        return repr(d[k]) if k in d else "(absent)"
    diffs = [f"{k}: saved {show(saved, k)}, now {show(config, k)}" for k in sorted(set(saved) | set(config))
             if k not in saved or k not in config or saved[k] != config[k]]
    if diffs:
        raise ValueError(f"{path} was written by a run with other settings; resuming it would not continue that run. "
                         f"Differing: " + "; ".join(diffs))


def find_state(output_dir, config: dict) -> Optional[dict]:
    """The training state in `output_dir`, loaded to the host and checked against `config`; None when there is none and
    `output_dir` holds no checkpoint.  ValueError for checkpoints without a state (a run that cannot be continued:
    training over it would overwrite its checkpoints), an unreadable state, another format version or another config."""
    output_dir = Path(output_dir)
    path = output_dir / STATE_NAME
    if not path.exists():
        ckpts = sorted(p.name for p in output_dir.glob("ckpt-*")) if output_dir.is_dir() else []
        if ckpts:
            raise ValueError(f"{output_dir} holds checkpoints ({', '.join(ckpts[:3])}{', ...' if len(ckpts) > 3 else ''}) "
                             f"but no {STATE_NAME}: that run cannot be continued; pass another output_dir or "
                             "resumable=False")
        return None
    try:
        state = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:
        raise ValueError(f"{path} is not a readable training state: {e}") from e
    if not isinstance(state, dict) or state.get("version") != STATE_VERSION:
        version = state.get("version") if isinstance(state, dict) else None
        raise ValueError(f"{path} has format version {version!r}, this build reads version {STATE_VERSION}")
    check_config(state["config"], config, path)
    return state


def _host_copy(obj):
    """`obj` with every tensor copied to the host (a fresh tensor, never an alias of a live one)."""
    if isinstance(obj, torch.Tensor):
        return obj.detach().to("cpu", copy=True)
    if isinstance(obj, dict):
        return {k: _host_copy(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_host_copy(v) for v in obj)
    return obj


def build_state(epoch: int, global_step: int, model, optimizer, scheduler, generator, train_losses, grad_norms,
                config: dict) -> dict:
    """The training state after epoch `epoch` (see the module docstring), every tensor on the host.  grad_norms: None
    without clipping."""
    state = dict(version=STATE_VERSION, epoch=int(epoch), global_step=int(global_step),
                 model=_host_copy(model.state_dict()), optimizer=_host_copy(optimizer.state_dict()),
                 scheduler=_host_copy(scheduler.state_dict()), rng="global" if generator is None else "generator",
                 rng_state=torch.get_rng_state() if generator is None else generator.get_state(),
                 train_losses=[float(v) for v in train_losses], config=dict(config))
    if grad_norms is not None:
        state["grad_norms"] = [float(v) for v in grad_norms]
    return state


def write_state(state: dict, output_dir) -> Path:
    """Write `state` to output_dir / STATE_NAME atomically: torch.save into a temporary file in output_dir, flushed to
    disk, then os.replace.  A write that fails or is killed leaves the previous state as it was."""
    output_dir = Path(output_dir)
    path = output_dir / STATE_NAME
    fd, tmp = tempfile.mkstemp(dir=output_dir, prefix=f".{STATE_NAME}.", suffix=".tmp")
    try:
        with os.fdopen(fd, "wb") as f:
            torch.save(state, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    return path


def restore_rng(state: dict, generator) -> None:
    """Set the visiting order's RNG (`generator`, or the global one for None) to the state's."""
    if generator is None:
        torch.set_rng_state(state["rng_state"])
    else:
        generator.set_state(state["rng_state"])
