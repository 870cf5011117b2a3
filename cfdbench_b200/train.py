"""`train_auto`: the reference's training loop (src/train_auto.py:181-313, `train`) with every step replayed from a CUDA
graph and one synchronisation per epoch.

The reference builds an autograd graph per batch, makes about fifteen native launches through ctypes around it and ends
every step with `loss["nmse"].item()`, so the host never runs ahead of the GPU.  Here one training step -- stage the
batch's indices, gather, pack the weights, training forward, loss forward and backward, backward, Adam, log the loss --
is captured once as a CUDA graph (plus one for a ragged last batch) and replayed once per step.  What changes from step
to step lives on the device and is read through a step cursor: the epoch's permutation, a table of Adam's bias-corrected
coefficients and the epoch's loss log.  Per epoch the host uploads the permutation and the table (asynchronously, from
pinned memory), resets the cursor, replays the graphs and copies the log back: that copy is the epoch's one
synchronisation.  The result is bit-identical to the eager loop `DeviceFrames.loader` + `model(**batch)` +
`loss["nmse"].backward()` + `FusedAdam.step()` + `zero_grad()` with the same generator and StepLR.

    from cfdbench_b200 import train_auto
    train_auto(model, train_data, dev_data, output_dir, num_epochs=..., lr=..., batch_size=...)   # for train(...)
    train_auto(..., rollout_steps=4)   # trained through 4-step rollouts of the model's own predictions
    train_auto(..., rollout_steps=4, rollout_grad_steps=1)   # pushforward: 3 steps without gradient, the 4th trained
    train_auto(..., rollout_steps=4, rollout_grad_steps=1, random_unroll=True)   # ... 0 to 3 of them, drawn per step
    train_auto(..., input_noise_std=0.01, noise_seed=1)      # Gaussian noise on every step's input frame
    train_auto(..., rollout_steps=4, input_noise_std=0.01, noise_every_step=True)   # ... and on every rollout step's
    train_auto(..., rollout_steps=4, teacher_forcing=[1 - e / 99 for e in range(100)], num_epochs=100)   # scheduled sampling
    train_auto(..., resumable=True)   # relaunching the same call continues an interrupted run bit for bit
"""
from __future__ import annotations

import ctypes as C
import json
import time
import warnings
from pathlib import Path
from shutil import copyfile
from typing import List, Optional

import numpy as np
import torch

from . import _lib, resume
from .data import (DeviceFrames, _check_chain, _check_split, _gather, _positive_int, as_device_frames, check_noise_args,
                   check_teacher_prob, index_batches, split_windows)
from .fno2d import capture_graph, side_stream
from .metrics import _evaluate_rollout, evaluate_auto
from .optim import FusedAdam

LOG_COLUMNS = ("mse", "rmse", "mae", "nmse", "mean_l2")   # one row of the epoch log: fno_loss_fwd's five scalars


# ------------------------------------------------------------------------------------------------ visiting order
def epoch_permutation(n: int, batch_size: int, generator=None) -> np.ndarray:
    """The sample order of one pass of `DataLoader(train_data, batch_size, shuffle=True, generator=generator)` (int64),
    drawing from the RNG exactly what that pass draws (`index_batches`)."""
    # the pass runs to its end: exhausting the sampler draws from an explicit generator too
    return np.asarray([i for b in index_batches(n, batch_size, True, generator) for i in b], dtype=np.int64)


def dev_eval_draw(generator=None) -> None:
    """What iterating the reference's `evaluate` loader (`DataLoader(dev_data, shuffle=False)`, src/train_auto.py:72-74)
    draws from the RNG: one base seed.  Without it every epoch after the first evaluation would be visited in another
    order than the reference's."""
    next(index_batches(1, 1, False, generator))


def index_stream(n: int, batch_size: int, num_epochs: int, eval_interval: int, generator=None,
                 start_epoch: int = 0) -> List[np.ndarray]:
    """The per-epoch sample orders `train_auto` visits in epochs start_epoch .. num_epochs - 1, consuming the RNG as
    `train_auto` does: epoch ep's permutation, then one evaluation draw when (ep + 1) % eval_interval == 0.  A resumed
    run starts at the epoch after its state's, with the RNG restored to where that epoch left it."""
    out = []
    for ep in range(start_epoch, num_epochs):
        out.append(epoch_permutation(n, batch_size, generator))
        if (ep + 1) % eval_interval == 0:
            dev_eval_draw(generator)
    return out


def unroll_lengths(unroll_seed: int, first_step: int, n: int, max_prefix: int) -> np.ndarray:
    """The prefix lengths `train_auto(random_unroll=True)` draws for Adam's 1-based steps first_step ..
    first_step + n - 1 (int64): step t runs `np.random.default_rng((unroll_seed, t)).integers(0, max_prefix + 1)`
    inference steps before its trained ones.  A pure function of (unroll_seed, t, max_prefix), so a resumed run draws
    what the uninterrupted one drew, whatever the epochs and batches."""
    return np.asarray([np.random.default_rng((unroll_seed, t)).integers(0, max_prefix + 1)
                       for t in range(first_step, first_step + n)], dtype=np.int64)


def dump_json(data, path) -> None:   # reference src/utils/common.py:23-25
    with open(path, "w", encoding="utf8") as f:
        json.dump(data, f, indent=2, ensure_ascii=False)


# ------------------------------------------------------------------------------------------------ the step graphs
class _StepGraphs:
    """The captured training step of a full batch of `batch_size` samples and, when n % batch_size != 0, of the ragged
    last batch.  Both graphs run on one set of static buffers sized for min(batch_size, n) samples: the ragged graph
    uses the first r samples' worth of every buffer.  The parameters and the optimizer state are read and written in
    place; the packed weight images are rebuilt inside the graph from the parameters as the previous replay's Adam
    left them."""
    teacher = False   # _RolloutStepGraphs with teacher forcing: flags drawn on the device from Adam's step

    def __init__(self, model, frames: DeviceFrames, batch_size: int, optimizer, n: Optional[int] = None,
                 noise_std: float = 0.0, noise_seed: int = 0):
        """n: the length of an epoch's permutation (default: every sample).  noise_std > 0: every step adds
        fno_add_input_noise(noise_std, noise_seed, step = Adam's 1-based step) to its input frames after the gather."""
        lib = self.lib = _lib.load()
        self.noise_std, self.noise_seed = noise_std, noise_seed
        self.model, self.frames, self.optimizer = model, frames, optimizer
        dev = self.dev = model.device
        n, gh, gw = frames.n if n is None else n, frames.height, frames.width
        self.n, self.gh, self.gw, self.stride = n, gh, gw, batch_size
        self.route = route = model._route(gh, gw)
        bmax = min(batch_size, n)
        n_full, rem = divmod(n, batch_size)
        self.sizes = [batch_size] * (n_full > 0) + [rem] * (rem > 0)   # the batch size of each graph
        self.counts = [n_full] * (n_full > 0) + [1] * (rem > 0)      # replays of each graph per epoch
        self.steps = n_full + (rem > 0)
        p = frames.n_case_params

        pk = model._pack(need_bwd=True)
        self.sw = model._static_weights(pk, gh, gw)   # graph-owned weight images, refilled by every replay
        model._refresh_static_weights(self.sw, pk, gh, gw)   # (also fills the coordinate tables)
        self.ws, self.ws_bufs = model._workspace(bmax, route)
        self.ts = model._train_state(bmax, route)
        self.flat, _, self.grads = model._grad_buffers()

        self.io = self._make_io(bmax, gh, gw, p)
        # FusedAdam(max_grad_norm=...): the step's global norm and clip coefficient, the epoch's norm log;
        # FusedAdam(ema_decay=...): the epoch's table of EMA decays, read by the cursor as the Adam coefficients are
        self.max_grad_norm, self.ema_decay = optimizer.max_grad_norm, optimizer.ema_decay
        if self.max_grad_norm is not None:
            self.io.update(norm=torch.empty(2, dtype=torch.float32, device=dev),
                           norm_log=torch.empty(self.steps, dtype=torch.float32, device=dev),
                           norm_scratch=torch.zeros((lib.fno_grad_norm_scratch_bytes() + 7) // 8, dtype=torch.float64,
                                                    device=dev))
            self.norm_host = torch.empty(self.steps, dtype=torch.float32, pin_memory=True)
        if self.ema_decay is not None:
            self.io["ema_d"] = torch.empty(self.steps, dtype=torch.float32, device=dev)
            self.ema_host = torch.empty(self.steps, dtype=torch.float32, pin_memory=True)
        self.uses_step = noise_std > 0 or self.teacher
        if self.uses_step:   # the epoch's first Adam step; a step's noise (and flag) step is this plus the cursor
            self.io["step_base"] = torch.zeros(1, dtype=torch.int64, device=dev)
            self.step_base_host = torch.empty(1, dtype=torch.int64, pin_memory=True)
        self.perm_host = torch.empty(n, dtype=torch.int64, pin_memory=True)
        self.coef_host = torch.empty(self.steps, 2, dtype=torch.float32, pin_memory=True)

        # Adam over the parameters that require grad (the ones autograd gives a .grad, so the ones FusedAdam.step
        # updates), in FusedAdam.step's tables; the state is created as FusedAdam creates it.  The backward writes every
        # parameter's gradient into the flat buffer; a frozen parameter's is not read.
        group = optimizer.param_groups[0]
        layout = [ent for ent in model._grad_layout()[0] if ent[1].requires_grad]
        self.params = [prm for _, prm, _, _ in layout]
        self.states = [optimizer.init_state(prm) for prm in self.params]
        self.adam = FusedAdam._tables(self.params, [self.flat[off:off + numel] for _, _, off, numel in layout],
                                      self.states, self.ema_decay is not None)
        self.adam_arr = (_lib.FnoAdamTensors * len(self.adam))(*self.adam)   # the norm launch's tables
        self.betas, self.eps, self.weight_decay = group["betas"], group["eps"], group["weight_decay"]

        with torch.no_grad(), side_stream(dev):
            self.graphs = self._capture()

    def _capture(self) -> list:
        """A warm-up of every launch except Adam and the log (it updates nothing: parameters, optimizer state and cursor
        stay as they are), then one capture per batch size."""
        for b in self.sizes:
            self._issue(b, update=False)
        return [capture_graph(lambda b=b: self._issue(b, update=True)) for b in self.sizes]

    def _replay(self, first_step: int) -> None:
        """The epoch's replays: each graph `count` times, in the order of `sizes`."""
        for g, count in zip(self.graphs, self.counts):
            for _ in range(count):
                g.replay()

    def _make_io(self, bmax: int, gh: int, gw: int, p: int) -> dict:
        """The static buffers of the step graphs."""
        lib, dev, n = self.lib, self.dev, self.n
        f32 = dict(dtype=torch.float32, device=dev)
        io = dict(
            perm=torch.zeros(n, dtype=torch.int64, device=dev),
            idx=torch.zeros(bmax, dtype=torch.int64, device=dev),
            inputs=torch.empty(bmax, 2, gh, gw, **f32), label=torch.empty(bmax, 2, gh, gw, **f32),
            mask=torch.empty(bmax, 1, gh, gw, **f32), cp=torch.empty(bmax, p, **f32),
            labm=torch.empty(bmax, 2, gh, gw, **f32), preds=torch.empty(bmax, 2, gh, gw, **f32),
            dpreds=torch.empty(bmax, 2, gh, gw, **f32), loss=torch.empty(5, **f32),
            scratch=torch.zeros(lib.fno_loss_scratch_bytes(), dtype=torch.uint8, device=dev),
            gout=torch.zeros(4, **f32),   # d/d(mse, rmse, mae, nmse) of loss["nmse"]: (0, 0, 0, 1)
            cursor=torch.zeros(1, dtype=torch.int32, device=dev),
            coef=torch.empty(self.steps, 2, **f32), log=torch.empty(self.steps, len(LOG_COLUMNS), **f32))
        io["gout"][3:].fill_(1.0)   # a fill kernel: assigning a Python number to a CUDA element is a blocking copy
        return io

    def _issue(self, b: int, update: bool) -> None:
        """One training step of batch b on the static buffers, on the current stream."""
        lib, io, sw, route = self.lib, self.io, self.sw, self.route
        st = C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)
        self._stage_indices(b, st)
        _gather(self.frames, io["idx"], b, io["inputs"], io["label"], io["mask"], io["cp"], st)
        self._add_noise(b, st)
        self._repack(st)
        inputs, mask, cp = io["inputs"][:b], io["mask"][:b], io["cp"][:b]
        preds, labm, dpreds = io["preds"][:b], io["labm"][:b], io["dpreds"][:b]
        torch.mul(io["label"][:b], mask, out=labm)   # Fno2d.forward's label * mask
        ts, ws = self.ts, self.ws
        route.call("forward_train", C.byref(sw["struct"]), inputs.data_ptr(), mask.data_ptr(), cp.data_ptr(),
                   preds.data_ptr(), C.byref(ts["sv"]), C.byref(ws), b, st)
        n_el = preds.numel()
        _lib.check(lib.fno_loss_fwd(preds.data_ptr(), labm.data_ptr(), n_el, io["scratch"].data_ptr(), io["loss"].data_ptr(),
                                    st), "fno_loss_fwd")
        _lib.check(lib.fno_loss_bwd(preds.data_ptr(), labm.data_ptr(), io["loss"].data_ptr(), io["gout"].data_ptr(),
                                    dpreds.data_ptr(), n_el, st), "fno_loss_bwd")
        route.call("backward", C.byref(sw["struct"]), C.byref(sw["struct_bwd"]), inputs.data_ptr(), mask.data_ptr(),
                   cp.data_ptr(), dpreds.data_ptr(), C.byref(ts["sv"]), C.byref(self.grads), C.byref(ts["sc"]),
                   C.byref(ws), None, None, b, st)
        if update:
            self._adam_and_log(io["loss"].data_ptr(), st)

    def _stage_indices(self, b: int, st) -> None:
        io = self.io
        _lib.check(self.lib.fno_train_stage_indices(io["perm"].data_ptr(), self.n, self.stride, b, io["cursor"].data_ptr(),
                                                    io["idx"].data_ptr(), st), "fno_train_stage_indices")

    def _add_noise(self, b: int, st) -> None:
        """The input noise of the gathered batch (nothing when noise_std is 0): step = step_base + cursor."""
        if self.noise_std > 0:
            io = self.io
            _lib.check(self.lib.fno_add_input_noise(io["inputs"].data_ptr(), io["mask"].data_ptr(), io["idx"].data_ptr(), b,
                                                    self.gh, self.gw, self.noise_std, self.noise_seed,
                                                    io["step_base"].data_ptr(), io["cursor"].data_ptr(), st),
                       "fno_add_input_noise")

    def _repack(self, st) -> None:
        """The packed weights, from the parameters as the previous step's Adam left them (Fno2d._pack's images)."""
        lib, model, sw = self.lib, self.model, self.sw
        L = model.num_layers
        wk, w0t, wkT = sw["dst"][:L], sw["dst"][L:2 * L], sw["dst"][2 * L:3 * L]
        for l, blk in enumerate(model.blocks):
            for dst, conj in ((wk[l], 0), (wkT[l], 1)):
                _lib.check(lib.fno_pack_mix_operand_from_weights(blk.conv0.weights1.data_ptr(),
                                                                 blk.conv0.weights2.data_ptr(), dst.data_ptr(), conj, st),
                           "fno_pack_mix_operand_from_weights")
            w0t[l].copy_(blk.w0.weight.view(w0t[l].shape).t())

    def _adam_and_log(self, loss_row: int, st) -> None:
        """Adam on the flat gradients, then the step's five loss scalars (at device address loss_row) into the log."""
        lib, io = self.lib, self.io
        b1, b2 = self.betas
        clip = None
        if self.max_grad_norm is not None:   # the global norm into its log row
            _lib.check(lib.fno_grad_norm(self.adam_arr, len(self.adam), self.max_grad_norm, io["norm"].data_ptr(),
                                         io["norm_scratch"].data_ptr(), io["norm_log"].data_ptr(), self.steps,
                                         io["cursor"].data_ptr(), st), "fno_grad_norm")
            clip = io["norm"][1:].data_ptr()
        ema_d = io["ema_d"].data_ptr() if self.ema_decay is not None else None
        for t in self.adam:
            _lib.check(lib.fno_adam_step_dev_ex(C.byref(t), io["coef"].data_ptr(), self.steps, io["cursor"].data_ptr(),
                                                b1, b2, self.eps, self.weight_decay, clip, t.ema, ema_d, st),
                       "fno_adam_step_dev_ex")
        _lib.check(lib.fno_train_log_step(loss_row, io["log"].data_ptr(), self.steps, io["cursor"].data_ptr(), st),
                   "fno_train_log_step")

    def epoch(self, perm: np.ndarray, lr: float, first_step: int) -> np.ndarray:
        """Train one epoch visiting the samples in `perm` at learning rate `lr`, Adam's 1-based step count starting at
        `first_step`.  Returns the (steps, 5) float32 log of fno_loss_fwd's scalars per step (LOG_COLUMNS); with
        clipping, `self.norms` then holds the (steps,) float32 pre-clip gradient norms."""
        io = self.io
        self.perm_host.numpy()[:] = perm   # the previous epoch's uploads completed before its log came back
        b1, b2 = self.betas
        _lib.check(self.lib.fno_adam_coefficients(lr, b1, b2, first_step, self.steps, self.coef_host.data_ptr()),
                   "fno_adam_coefficients")
        io["perm"].copy_(self.perm_host, non_blocking=True)
        io["coef"].copy_(self.coef_host, non_blocking=True)
        if self.ema_decay is not None:
            _lib.check(self.lib.fno_ema_decays(self.ema_decay, first_step, self.steps, self.ema_host.data_ptr()),
                       "fno_ema_decays")
            io["ema_d"].copy_(self.ema_host, non_blocking=True)
        if self.uses_step:
            self.step_base_host[0] = first_step
            io["step_base"].copy_(self.step_base_host, non_blocking=True)
        io["cursor"].zero_()
        self._replay(first_step)
        if self.max_grad_norm is not None:   # complete once the log below has come back
            self.norm_host.copy_(io["norm_log"], non_blocking=True)
        log = io["log"].cpu().numpy()   # the epoch's one synchronisation
        if self.max_grad_norm is not None:
            self.norms = self.norm_host.numpy().copy()
            self.optimizer.last_grad_norm = io["norm"][0].clone()
        # the state torch.optim.Adam would hold, and the version bump FusedAdam.step makes (Fno2d's packed-weight cache
        # and inference graphs are keyed on the parameters' versions)
        for st in self.states:
            st["step"] += self.steps
        for prm in self.params:
            torch.autograd.graph.increment_version(prm)
        return log


class _RolloutStepGraphs(_StepGraphs):
    """The captured step of training through `k`-step rollouts (train_auto with rollout_steps = k > 1): the epoch's
    permutation holds window starts, and a step is stage indices -> gather window (inputs, mask and case parameters of
    the start sample, the k masked targets) -> [input noise] -> weight repack -> [pushforward prefix] -> rollout
    training forward into one reused saved set -> K-step loss forward and backward -> rollout backward (one recomputing
    sweep, no input gradients) into the flat gradient buffer -> Adam -> log of the aggregate loss row.  Same graphs,
    buffers-per-batch layout and epoch as _StepGraphs; the per-step buffers are [k][b] blocks of the first k*b samples'
    worth of (k, bmax, ...) buffers.

    grad_steps = g < k (pushforward): the first k - g steps run without gradient through the inference rollout
    (fno_[grid_]rollout, the kernels generate_many runs) into a (k - g, bmax, ...) prefix buffer, on the step's
    workspace (the model's inference workspace for bmax samples, with the bf16 ym_img image); the training rollout, the
    loss against targets k - g ... k - 1 and the backward then cover the last g steps from the prefix's last frame.

    noise_every_step (with noise_std > 0): rollout step s of the window (prefix and trained steps alike) is fed its
    input plus the noise of stream s (the start frame keeps the gather's stream-0 noise).  The prefix and the trained
    steps run the *_noise drivers with k0 = 0 and k0 = k - g, writing the perturbed frames into (k - g, bmax, ...) and
    (g, bmax, ...) fed-frame buffers: k more frames per sample than without, and one more launch per rollout step.

    random_unroll (g < k): Adam's step t runs u_t = unroll_lengths(unroll_seed, t, 1, k - g)[0] prefix steps instead of
    k - g, and trains steps u_t .. u_t + g - 1 of the window (u_t = 0: no prefix launch, the start frame is trained).
    One step is captured per u in 0 .. k - g and batch size, every capture on the same buffers (the prefix buffer holds
    the longest prefix); the epoch replays the graph of each step's u_t.

    teacher (g = k, scheduled sampling): after the gather, fno_teacher_flags draws the (k - 1, b) flags of the step
    from the epoch's probability (a device float uploaded with the epoch's tables) and step = step_base + cursor; the
    training forward and the sweep are the *_feed drivers, fed the gathered targets 0 .. k - 2 as the true frames.  A
    (k, bmax, ...) fed-frame buffer and one more launch per rollout step, as every-step noise."""

    def __init__(self, model, frames: DeviceFrames, batch_size: int, optimizer, n_windows: int, steps: int,
                 time_step_size: int, grad_steps: Optional[int] = None, noise_std: float = 0.0, noise_seed: int = 0,
                 noise_every_step: bool = False, random_unroll: bool = False, unroll_seed: int = 0,
                 teacher: bool = False, teacher_seed: int = 0):
        self.k, self.tss = steps, time_step_size
        self.g = steps if grad_steps is None else grad_steps
        self.every = noise_every_step and noise_std > 0
        self.random_unroll, self.unroll_seed = random_unroll, unroll_seed
        self.teacher, self.teacher_seed = teacher, teacher_seed
        if teacher:
            assert self.g == steps > 1 and not random_unroll
            self.prob_host = torch.zeros(1, dtype=torch.float32, pin_memory=True)
        super().__init__(model, frames, batch_size, optimizer, n=n_windows, noise_std=noise_std, noise_seed=noise_seed)

    def _make_io(self, bmax: int, gh: int, gw: int, p: int) -> dict:
        lib, dev, n, k, g = self.lib, self.dev, self.n, self.k, self.g
        f32 = dict(dtype=torch.float32, device=dev)
        io = dict(
            perm=torch.zeros(n, dtype=torch.int64, device=dev),
            idx=torch.zeros(bmax, dtype=torch.int64, device=dev),
            inputs=torch.empty(bmax, 2, gh, gw, **f32), mask=torch.empty(bmax, 1, gh, gw, **f32),
            cp=torch.empty(bmax, p, **f32), labels=torch.empty(k, bmax, 2, gh, gw, **f32),
            preds=torch.empty(g, bmax, 2, gh, gw, **f32), dpreds=torch.empty(g, bmax, 2, gh, gw, **f32),
            carry=torch.empty(bmax, 2, gh, gw, **f32), loss=torch.empty(g + 1, 5, **f32),
            scratch=torch.zeros(lib.fno_loss_seq_scratch_bytes(g), dtype=torch.uint8, device=dev),
            gout=torch.zeros(4, **f32),   # d/d(mse, rmse, mae, nmse) of the aggregate's nmse: (0, 0, 0, 1)
            cursor=torch.zeros(1, dtype=torch.int32, device=dev),
            coef=torch.empty(self.steps, 2, **f32), log=torch.empty(self.steps, len(LOG_COLUMNS), **f32))
        if g < k:
            io["prefix"] = torch.empty(k - g, bmax, 2, gh, gw, **f32)
        if self.every or self.teacher:
            io["fed"] = torch.empty(g, bmax, 2, gh, gw, **f32)
        if self.every and g < k:
            io["fed_prefix"] = torch.empty(k - g, bmax, 2, gh, gw, **f32)
        if self.teacher:
            io["flags"] = torch.zeros(k - 1, bmax, dtype=torch.uint8, device=dev)
            io["prob"] = torch.zeros(1, **f32)
        io["gout"][3:].fill_(1.0)
        return io

    def _teacher(self):
        """The fno_teacher of the step: the gathered targets 0 .. k - 2 and the step's flags, [k - 1][b] blocks."""
        io = self.io
        return C.byref(_lib.FnoTeacher(io["labels"].data_ptr(), io["flags"].data_ptr()))

    def epoch(self, perm: np.ndarray, lr: float, first_step: int, teacher_prob: float = 0.0) -> np.ndarray:
        """_StepGraphs.epoch; with teacher forcing the epoch's flags are drawn with probability `teacher_prob`."""
        if self.teacher:   # the previous epoch's upload completed before its log came back
            self.prob_host[0] = teacher_prob
            self.io["prob"].copy_(self.prob_host, non_blocking=True)
        return super().epoch(perm, lr, first_step)

    def _noise(self, k0: int):
        """The fno_noise of the step's rollout calls whose first step is window step k0: step = step_base + cursor,
        as the start frame's noise."""
        io = self.io
        return C.byref(_lib.FnoNoise(self.noise_std, self.noise_seed, io["idx"].data_ptr(), io["step_base"].data_ptr(),
                                     io["cursor"].data_ptr(), k0))

    def _capture(self) -> list:
        """Without random_unroll, _StepGraphs' graphs; with it, graphs[u][i]: prefix length u, batch size sizes[i]."""
        if not self.random_unroll:
            return super()._capture()
        us = range(self.k - self.g + 1)
        for u in us:
            for b in self.sizes:
                self._issue(b, update=False, u=u)
        return [[capture_graph(lambda b=b, u=u: self._issue(b, update=True, u=u)) for b in self.sizes] for u in us]

    def _replay(self, first_step: int) -> None:
        if not self.random_unroll:
            return super()._replay(first_step)
        # drawn step by step (about 30 us each), so that the host draws step t + 1 while the device runs step t
        t = first_step
        for i, count in enumerate(self.counts):
            for _ in range(count):
                self.graphs[int(unroll_lengths(self.unroll_seed, t, 1, self.k - self.g)[0])][i].replay()
                t += 1

    def _issue(self, b: int, update: bool, u: Optional[int] = None) -> None:
        """u: the prefix length (default k - g)."""
        lib, io, sw, route, k, g = self.lib, self.io, self.sw, self.route, self.k, self.g
        u = k - g if u is None else u
        st = C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)
        self._stage_indices(b, st)
        _gather(self.frames, io["idx"], b, io["inputs"], None, io["mask"], io["cp"], st,
                window=(k, self.tss, io["labels"]))
        self._add_noise(b, st)
        if self.teacher:
            _lib.check(lib.fno_teacher_flags(io["idx"].data_ptr(), b, k, io["prob"].data_ptr(), self.teacher_seed,
                                             io["step_base"].data_ptr(), io["cursor"].data_ptr(), io["flags"].data_ptr(),
                                             st), "fno_teacher_flags")
        self._repack(st)
        x, mk, cp = io["inputs"].data_ptr(), io["mask"].data_ptr(), io["cp"].data_ptr()
        preds, labels, dpreds = io["preds"].data_ptr(), io["labels"].data_ptr(), io["dpreds"].data_ptr()
        ts, ws = self.ts, self.ws
        n_el = b * 2 * self.gh * self.gw   # per step
        if u > 0:   # the pushforward prefix, without gradient; the trained steps start from its last frame
            pre = io["prefix"].data_ptr()
            if self.every:
                route.call("rollout_noise", C.byref(sw["struct"]), x, mk, cp, pre, u, C.byref(ws), self._noise(0),
                           io["fed_prefix"].data_ptr(), b, st)
            else:
                route.call("rollout", C.byref(sw["struct"]), x, mk, cp, pre, u, C.byref(ws), b, st)
            x = pre + (u - 1) * n_el * 4
            labels += u * n_el * 4
        if self.teacher:
            route.call("rollout_forward_train_feed", C.byref(sw["struct"]), x, mk, cp, preds, g, C.byref(ts["sv"]),
                       C.byref(ws), self._noise(u) if self.every else None, self._teacher(), io["fed"].data_ptr(), b, st)
        elif self.every:
            route.call("rollout_forward_train_noise", C.byref(sw["struct"]), x, mk, cp, preds, g, C.byref(ts["sv"]),
                       C.byref(ws), self._noise(u), io["fed"].data_ptr(), b, st)
        else:
            route.call("rollout_forward_train", C.byref(sw["struct"]), x, mk, cp, preds, g, C.byref(ts["sv"]),
                       C.byref(ws), b, st)
        _lib.check(lib.fno_loss_seq_fwd(preds, labels, n_el, g, io["scratch"].data_ptr(), io["loss"].data_ptr(), st),
                   "fno_loss_seq_fwd")
        _lib.check(lib.fno_loss_seq_bwd(preds, labels, io["loss"].data_ptr(), io["gout"].data_ptr(), dpreds, n_el, g, st),
                   "fno_loss_seq_bwd")
        if self.teacher:
            route.call("rollout_backward_feed", C.byref(sw["struct"]), C.byref(sw["struct_bwd"]), x, mk, cp, preds,
                       dpreds, g, C.byref(ts["sv"]), C.byref(self.grads), C.byref(ts["sc"]), C.byref(ws),
                       self._noise(u) if self.every else None, self._teacher(), io["fed"].data_ptr(),
                       io["carry"].data_ptr(), None, None, b, st)
        elif self.every:
            route.call("rollout_backward_noise", C.byref(sw["struct"]), C.byref(sw["struct_bwd"]), x, mk, cp, preds,
                       dpreds, g, C.byref(ts["sv"]), C.byref(self.grads), C.byref(ts["sc"]), C.byref(ws),
                       self._noise(u), io["fed"].data_ptr(), io["carry"].data_ptr(), None, None, b, st)
        else:
            route.call("rollout_backward", C.byref(sw["struct"]), C.byref(sw["struct_bwd"]), x, mk, cp, preds, dpreds,
                       g, C.byref(ts["sv"]), C.byref(self.grads), C.byref(ts["sc"]), C.byref(ws), io["carry"].data_ptr(),
                       None, None, b, st)
        if update:
            self._adam_and_log(io["loss"][g].data_ptr(), st)


# ------------------------------------------------------------------------------------------------ train_auto
def _teacher_record(teacher_forcing):
    """teacher_forcing as plain Python values for the resume record: a float, or a list of floats."""
    if isinstance(teacher_forcing, (int, float, np.integer, np.floating)):
        return float(teacher_forcing)
    return [float(v) for v in teacher_forcing]


def teacher_schedule(teacher_forcing, num_epochs: int, teacher_seed, rollout_steps: int, grad_steps: int,
                     random_unroll: bool) -> Optional[List[float]]:
    """The per-epoch teacher-forcing probabilities of `train_auto(teacher_forcing=..., teacher_seed=...)`: None when
    teacher forcing is off (None, or 0 in every epoch: the call runs what runs without it), else num_epochs floats.
    ValueError, naming the argument, for a value that is not a real in [0, 1], a sequence shorter than num_epochs, a
    teacher_seed that is not an int in [0, 2^64), or teacher forcing with rollout_steps = 1, pushforward
    (rollout_grad_steps < rollout_steps) or random_unroll."""
    if isinstance(teacher_seed, bool) or not isinstance(teacher_seed, (int, np.integer)) \
            or not 0 <= int(teacher_seed) < 2 ** 64:
        raise ValueError(f"teacher_seed must be an int in [0, 2^64), got {teacher_seed!r}")
    if teacher_forcing is None:
        return None
    if isinstance(teacher_forcing, (bool, str, bytes)):
        raise ValueError(f"teacher_forcing must be None, a real in [0, 1] or a sequence of them, got {teacher_forcing!r}")
    if isinstance(teacher_forcing, (int, float, np.integer, np.floating)):
        probs = [check_teacher_prob(teacher_forcing, "teacher_forcing")] * num_epochs
    else:
        try:
            values = list(teacher_forcing)
        except TypeError:
            raise ValueError(f"teacher_forcing must be None, a real in [0, 1] or a sequence of them, got "
                             f"{teacher_forcing!r}") from None
        if len(values) < num_epochs:
            raise ValueError(f"teacher_forcing has {len(values)} values, fewer than num_epochs={num_epochs} (one per "
                             "epoch)")
        probs = [check_teacher_prob(v, f"teacher_forcing[{i}]") for i, v in enumerate(values)][:num_epochs]
    if rollout_steps < 2:
        raise ValueError("teacher_forcing chooses what rollout steps 1 .. K - 1 are fed: it needs rollout_steps > 1")
    if grad_steps < rollout_steps or random_unroll:
        raise ValueError(f"teacher_forcing does not combine with pushforward training: it needs rollout_grad_steps = "
                         f"rollout_steps and random_unroll=False, got rollout_grad_steps={grad_steps}, "
                         f"random_unroll={random_unroll}")
    return probs if any(p > 0 for p in probs) else None


def _ema_shadow(model):
    """A Fno2d with `model`'s configuration, storage mode, device and kernel choices, holding a copy of its weights: the
    model the EMA weights are evaluated and saved through.  Built without drawing from the CPU RNG (the parameters'
    initialisation would shift the visiting order of a train_auto that uses the global RNG)."""
    from .fno2d import Fno2d
    with torch.random.fork_rng(devices=[]):
        shadow = Fno2d(model.in_chan, model.out_chan, model.n_case_params, model.loss_fn, model.num_layers,
                       modes1=model.modes1, modes2=model.modes2, hidden_dim=model.hidden_dim, act_dtype=model.act_dtype,
                       device=model.device)
    for name in ("graph_rollout", "fused_block", "max_graphs", "generic_grid_at_64"):
        setattr(shadow, name, getattr(model, name))
    shadow.load_state_dict(model.state_dict())
    return shadow


def train_auto(model, train_data, dev_data, output_dir, num_epochs: int = 400, lr: float = 1e-3, lr_step_size: int = 1,
               lr_gamma: float = 0.9, batch_size: int = 2, eval_batch_size: int = 2, log_interval: int = 10,
               eval_interval: int = 2, generator: Optional[torch.Generator] = None, rollout_steps: int = 1,
               time_step_size: Optional[int] = None, input_noise_std: float = 0.0, noise_seed: int = 0,
               rollout_grad_steps: Optional[int] = None, noise_every_step: bool = False,
               dev_rollout_steps: Optional[int] = None, max_grad_norm: Optional[float] = None,
               ema_decay: Optional[float] = None, resumable: bool = False, random_unroll: bool = False,
               unroll_seed: int = 0, teacher_forcing=None, teacher_seed: int = 0) -> dict:
    """What the reference's `train(model, train_data, dev_data, output_dir, ...)` does (src/train_auto.py:181-313), with
    its argument names and defaults, every training step replayed from a CUDA graph and one synchronisation per epoch.

    model: the drop-in `Fno2d` on a CUDA device, with a loss whose score names include "nmse" (the loss the reference
    backpropagates); the step computes that loss with the native MseLoss kernels.  train_data / dev_data: the
    reference's dataset objects or `DeviceFrames` of them (a dataset is uploaded once, in float32).

    - Optimizer: `FusedAdam(model.parameters(), lr)` with `torch.optim.lr_scheduler.StepLR(step_size=lr_step_size,
      gamma=lr_gamma)`; each epoch runs at the learning rate StepLR leaves in the parameter group.
    - Visiting order: the reference's for the same RNG -- `generator`, or the global RNG for None, as in the reference.
      Each epoch draws what one pass of `DataLoader(train_data, batch_size, shuffle=True)` draws, and each evaluation
      the one base seed that iterating the reference's `DataLoader(dev_data, shuffle=False)` draws.  The ragged last
      batch is kept (drop_last=False).
    - Every `eval_interval` epochs: `evaluate_auto(model, <DeviceFrames of dev_data>, batch_size=eval_batch_size)` and
      the reference's files in `output_dir / f"ckpt-{ep}"`: dev_scores.json, train_loss.json, model.pt (the previous
      one copied to backup_model.pt first when it exists) and scores.json (ep, train_loss, dev_loss, time).  At the end
      `output_dir / "train_losses.json"`.  JSON is written as the reference's dump_json writes it.
    - Logging: the reference's line every `log_interval` steps, printed at the end of the epoch from the device log, so
      its `time` field is the time of printing, not of the step.
    - Not reproduced: example.png, train_losses.png and the evaluation images; `measure_time`.
    - rollout_steps = K > 1 trains through K-step rollouts (`Fno2d.rollout`): each step of an epoch takes a batch of
      window starts j and trains on (nmse_0 + ... + nmse_{K-1}) / K, nmse_k = MseLoss(step k's prediction,
      labels[j + k s] * mask_j)["nmse"], s = time_step_size (default: train_data.time_step_size), every step masked with
      the start sample's mask.  The windows are `rollout_windows(case_ids, K, s)`, which never cross a case; each epoch
      visits a permutation of them that draws from the RNG what a DataLoader over that many samples draws.  The log and
      train_losses hold the aggregate (each column the mean over the K steps).  The split must chain
      (frames_in[j + k s] == frames_out[j + (k-1) s] for every pair a window uses): that is checked once on the device
      before training.  The dev evaluation stays single-step unless dev_rollout_steps is given (below).
      rollout_steps = 1 is the single-step loop above, launch for launch.
    - rollout_grad_steps = G (1 <= G <= K, default K) is pushforward training: of each window's K steps the first
      K - G run without gradient through the inference rollout (the kernels `generate_many` runs), and only the last
      G are trained, from the prefix's last frame, on (nmse_{K-G} + ... + nmse_{K-1}) / G; the log and train_losses
      hold that mean.  G = K is the full rollout above, launch for launch; with K = 1 only G = 1 is valid.
    - random_unroll=True (needs G < K) draws the prefix length per step, as Brandstetter, Worrall & Welling's
      pushforward trick does per batch: Adam's step t runs u_t = unroll_lengths(unroll_seed, t, 1, K - G)[0] inference
      steps (uniform in 0 .. K - G; u_t = 0 launches no prefix) and trains the G steps after them, from prefix frame
      u_t - 1 or the start frame, on (nmse_{u_t} + ... + nmse_{u_t+G-1}) / G.  The windows, the permutation and the
      draws from `generator` are those of the fixed-prefix call; u_t depends on (unroll_seed, t, K - G) only, an int
      >= 0 never drawn from `generator`.  One step graph is captured per prefix length, all on the same buffers.  With
      input noise the start frame is perturbed as above; with noise_every_step the prefix runs k0 = 0 over u_t steps
      and the trained steps k0 = u_t (window step k is fed noise stream k).  One step is bit-identical to the eager
      loop of the pushforward one with u = unroll_lengths(unroll_seed, t, 1, K - G)[0] in place of K - G (INTEGRATION
      §3).  False (the default) launches and replays exactly what runs without the option.
    - input_noise_std = sigma > 0 adds Gaussian noise to every step's (start) input frame where the mask is non-zero,
      `DeviceFrames.batch(..., noise_std=sigma, noise_seed=noise_seed, noise_step=t)` with t Adam's 1-based global step
      of that update.  The noise comes from a counter-based RNG seeded by `noise_seed` (an int in [0, 2^64)), never
      from `generator`, so the visiting order is the one without noise; 0 launches nothing extra.  One step is
      bit-identical to the eager loop

          b = frames.rollout_batch(idx, K, noise_std=sigma, noise_seed=noise_seed, noise_step=t)
          x = b["inputs"]
          if K > G:
              with torch.no_grad():
                  x = model.generate_many(x, b["case_params"], b["mask"], K - G)[-1]
          seq = model.rollout(x, b["case_params"], b["mask"], G)
          loss = sum(model.loss_fn(preds=seq[g], labels=b["labels"][K - G + g])["nmse"] for g in range(G)) / G

      (at K = 1: `frames.batch(idx, noise_std=...)` and the single-step loss).
    - noise_every_step=True (with input_noise_std > 0 and K > 1) perturbs the frame every rollout step is fed, not
      only the start frame: window step k >= 1 is fed its (clean) predecessor plus the noise of stream k,
      `add_input_noise(x, mask, idx, sigma, noise_seed, t, stream=k)`, in the pushforward prefix and in the trained
      steps alike.  Predictions and targets stay clean.  It costs one launch and one frame per sample per rollout
      step.  Without noise, or at K = 1, the flag changes nothing, launch for launch.  One step is bit-identical to
      the eager loop

          b = frames.rollout_batch(idx, K, noise_std=sigma, noise_seed=noise_seed, noise_step=t)
          ids = torch.as_tensor(idx, device=b["inputs"].device)
          x = b["inputs"]
          for k in range(K - G):
              if k > 0:
                  x = add_input_noise(x, b["mask"], ids, sigma, noise_seed, t, stream=k)
              with torch.no_grad():
                  x = model.generate_many(x, b["case_params"], b["mask"], 1)[0]
          seq = model.rollout(x, b["case_params"], b["mask"], G, noise=RolloutNoise(sigma, noise_seed, t, ids, K - G))
          loss = sum(model.loss_fn(preds=seq[g], labels=b["labels"][K - G + g])["nmse"] for g in range(G)) / G

    - teacher_forcing = p (a real in [0, 1], or a sequence of at least num_epochs of them, one per epoch) is scheduled
      sampling (Bengio et al. 2015) over the K-step window (needs K > 1 and no pushforward): rollout step s >= 1 of a
      window is fed the true frame, the masked target of step s - 1, with probability p, else the model's prediction
      of step s - 1.  The flags are drawn on the device per window and step from `teacher_seed` and Adam's step
      (`teacher_forcing_flags`); p reaches the device with each epoch's uploads.  The gradient through a forced step's
      input is cut: prediction s - 1 of a forced window gets the loss's gradient alone.  With noise_every_step the
      noise of stream s is added to whichever frame was chosen.  It costs one launch and one frame per sample per
      rollout step.  None, or p = 0 in every epoch, runs exactly what runs without it.  One step is bit-identical to
      the eager loop (p the epoch's value)

          b = frames.rollout_batch(idx, K, noise_std=sigma, noise_seed=noise_seed, noise_step=t)
          ids = torch.as_tensor(idx, device=b["inputs"].device)
          flags = teacher_forcing_flags(ids, K, p, teacher_seed, t)
          noise = RolloutNoise(sigma, noise_seed, t, ids, 0) if noise_every_step else None
          seq = model.rollout(b["inputs"], b["case_params"], b["mask"], K, noise=noise,
                              teacher=TeacherForcing(b["labels"][:K - 1], flags))
          loss = sum(model.loss_fn(preds=seq[k], labels=b["labels"][k])["nmse"] for k in range(K)) / K

    - dev_rollout_steps = S selects checkpoints by rollout error: every evaluation also runs
      `evaluate_rollout_auto(model, <DeviceFrames of dev_data>, S, time_step_size)` -- every S-step window of the dev
      split rolled out from its start sample, step k against the frame k + 1 time steps on -- writes its result to
      `ckpt-{ep}/dev_rollout_scores.json`, and writes scores.json with dev_loss = its `loss` (the mean over the S steps
      of the nmse) and dev_loss_single_step = the single-step dev_loss, so that the reference's get_best_ckpt /
      load_best_ckpt, which pick the lowest dev_loss, pick the checkpoint with the lowest rollout error.
      dev_scores.json stays the single-step evaluation.  The dev split's time step size is the time_step_size
      argument, else dev_data.time_step_size; it must have an S-step window and chain (checked once on the device
      before training).  The evaluation draws nothing from the RNG, so training is bit-identical with and without it;
      None (the default) runs exactly what runs without the option.
    - max_grad_norm = c clips the global gradient norm to c before every update, `clip_grad_norm_(every trainable
      parameter, c)`, inside the step graph: one float64 norm launch (bit-reproducible) and the coefficient read by the
      Adam launch.  Each step's pre-clip norm is logged on the device: the log line gains grad_norm, the result
      `grad_norms` (every step, every epoch) and `output_dir / "grad_norms.json"` holds them.
    - ema_decay = d keeps an exponential moving average of the weights, updated by the Adam launch: diffusers'
      EMAModel with warmup, decay min(d, 1 - t^(-3/4)) at Adam's step t (0 at t = 1: the EMA starts as the trained
      weights), inv_gamma 1, power 3/4, as train_diffusers.py configures it.  Every evaluation runs on an EMA copy of the
      model (same configuration, storage mode and device; `FusedAdam.copy_ema_to`), so dev_scores.json, scores.json's
      dev_loss (and the rollout score with dev_rollout_steps) and model.pt are the EMA weights', which the reference's
      load_best_ckpt and test_multistep then read.  `model` itself ends with the trained weights; the result gains
      `ema_model`.
      With either option one step is bit-identical to the eager loops above with
      `FusedAdam(model.parameters(), lr, max_grad_norm=max_grad_norm, ema_decay=ema_decay)`, its state["ema"] and
      `last_grad_norm` included.  None (the defaults) launches exactly what runs without the options.
    - resumable=True keeps the full training state in `output_dir / "training_state.pt"` (cfdbench_b200.resume): the
      trained weights, FusedAdam's state (step, both moments, the EMA), StepLR's, the visiting order's RNG state,
      Adam's global step, train_losses / grad_norms and a config record.  It is written atomically (a temporary file,
      then os.replace) after each evaluation epoch's checkpoint files and after the last epoch, one file overwritten
      each time.  At start-up an existing state is checked against this call (the model's configuration, every
      argument that changes the trajectory or the checkpoint scores, and each split's size, grid, case-parameter count,
      frame dtype and case_ids hash -- not the frame contents; num_epochs and log_interval may change), loaded into
      `model` and the new optimizer, scheduler and RNG, and training continues from the epoch after the one it records,
      bit-identical to a run that was never interrupted; its train_losses / grad_norms cover the whole run.  With
      num_epochs no larger than the epochs already trained no step runs and the finished run's result is returned
      (the JSON files rewritten); a larger num_epochs extends the run, equal to a longer straight run.  Without a state
      an output_dir that holds ckpt-* directories is refused, and otherwise the run starts fresh.  So relaunching the
      same call is the whole recovery procedure; a killed run retrains at most the epochs since the last evaluation.
      False (the default) writes and reads nothing more than without the option.
    Returns dict(train_losses=[per-step nmse, every epoch], optimizer=the FusedAdam, start_epoch=the first epoch this
    call trained: 0, or E + 1 after resuming from epoch E).  Its state holds the true step
    count (its state_dict loads into torch.optim.Adam), and the parameters' version counters are bumped, so the
    model's packed weights and inference graphs are rebuilt on the next call.  Raises before any device work on: a
    model that is not the drop-in Fno2d, a CPU model (FnoNativeError), a loss without "nmse", non-positive sizes,
    intervals or epoch count, a model whose parameters are all frozen, an empty or malformed split, a split whose
    case-parameter count differs from the model's, data parallel enabled, or a grid / storage mode the model rejects;
    and, as ValueError before any training step, a non-positive rollout_steps or time_step_size, rollout_steps > 1 with
    no time_step_size, a split without a single K-step window, or a split whose frames do not chain.  Also raises
    ValueError before any device work for an input_noise_std that is negative, NaN, infinite or not a real number, a
    noise_seed that is not an int in [0, 2^64), a rollout_grad_steps that is not an int in 1..rollout_steps, a
    noise_every_step that is not a bool, a dev_rollout_steps that is not None or a positive int, a max_grad_norm
    that is not None or a finite real > 0, or an ema_decay that is not None or a real in [0, 1); with
    dev_rollout_steps, as ValueError before any training step, a dev split without a time step size, without a single
    S-step window, or whose frames do not chain.  With resumable=True, also ValueError before any device work for a
    training_state.pt that does not load, has another format version or was written with another config (naming every
    differing field), or for an output_dir with ckpt-* directories and no training_state.pt; ValueError for a
    resumable that is not a bool; for a random_unroll that is not a bool, an unroll_seed that is not an int >= 0, or
    random_unroll=True with rollout_steps = 1 or rollout_grad_steps = rollout_steps; for a teacher_forcing that is not
    None, a real in [0, 1] or a sequence of at least num_epochs of them, a teacher_seed that is not an int in
    [0, 2^64), or teacher_forcing with rollout_steps = 1, rollout_grad_steps < rollout_steps or random_unroll.
    Frozen parameters (requires_grad=False) are not updated, as FusedAdam.step skips them.  Data parallel training in
    this loop is not supported."""
    from .fno2d import Fno2d
    from .optim import FusedAdam, check_stabiliser_args
    if not isinstance(model, Fno2d):
        raise TypeError(f"train_auto runs the drop-in cfdbench_b200.Fno2d, got {type(model).__name__}")
    names = list(model.loss_fn.get_score_names())
    if "nmse" not in names:
        raise ValueError(f"the model's loss has scores {names}: train_auto backpropagates loss['nmse'], as the reference")
    for name, v in (("num_epochs", num_epochs), ("lr_step_size", lr_step_size), ("batch_size", batch_size),
                    ("eval_batch_size", eval_batch_size), ("log_interval", log_interval), ("eval_interval", eval_interval),
                    ("rollout_steps", rollout_steps)):
        _positive_int(name, v)
    input_noise_std = check_noise_args(input_noise_std, noise_seed, std_name="input_noise_std")
    if not isinstance(noise_every_step, bool):
        raise ValueError(f"noise_every_step must be a bool, got {noise_every_step!r}")
    if not isinstance(resumable, bool):
        raise ValueError(f"resumable must be a bool, got {resumable!r}")
    if dev_rollout_steps is not None:
        dev_rollout_steps = _positive_int("dev_rollout_steps", dev_rollout_steps)
    max_grad_norm, ema_decay = check_stabiliser_args(max_grad_norm, ema_decay)
    grad_steps = rollout_steps if rollout_grad_steps is None else rollout_grad_steps
    if isinstance(grad_steps, bool) or not isinstance(grad_steps, (int, np.integer)) or not 1 <= grad_steps <= rollout_steps:
        raise ValueError(f"rollout_grad_steps must be an int in 1..rollout_steps={rollout_steps}, got {rollout_grad_steps!r}")
    grad_steps = int(grad_steps)
    if not isinstance(random_unroll, bool):
        raise ValueError(f"random_unroll must be a bool, got {random_unroll!r}")
    if isinstance(unroll_seed, bool) or not isinstance(unroll_seed, (int, np.integer)) or unroll_seed < 0:
        raise ValueError(f"unroll_seed must be a non-negative int, got {unroll_seed!r}")
    if random_unroll and not grad_steps < rollout_steps:
        raise ValueError(f"random_unroll draws the pushforward prefix length: it needs rollout_steps > 1 and "
                         f"rollout_grad_steps < rollout_steps, got rollout_steps={rollout_steps}, "
                         f"rollout_grad_steps={rollout_grad_steps!r}")
    teacher_probs = teacher_schedule(teacher_forcing, num_epochs, teacher_seed, rollout_steps, grad_steps, random_unroll)
    if model._dp_enabled:
        raise ValueError("train_auto does not run data parallel: its step graph has no all-reduce")
    if not any(p.requires_grad for p in model.parameters()):
        raise ValueError("every parameter of the model is frozen: there is nothing to train")
    dev = model.device
    train_split = _check_split(model, train_data, "train_data")
    dev_split = _check_split(model, dev_data, "dev_data")
    windows = tss = None   # rollout_steps > 1: the window starts of the train split and their time step size
    if rollout_steps > 1:
        windows, tss = split_windows(train_split, rollout_steps, time_step_size, "train_data", "rollout_steps")
    elif time_step_size is not None:
        _positive_int("time_step_size", time_step_size)
    dev_windows = dev_tss = None   # dev_rollout_steps = S: the window starts of the dev split, likewise
    if dev_rollout_steps is not None:
        dev_windows, dev_tss = split_windows(dev_split, dev_rollout_steps, time_step_size, "dev_data", "dev_rollout_steps")
    state = config = None
    if resumable:
        # Python floats, so that StepLR's decay of a restored learning rate runs in the same arithmetic as a straight
        # run's, and the state holds no numpy scalar (it must load with weights_only=True)
        lr, lr_gamma = float(lr), float(lr_gamma)
        config = resume.run_config(
            model, train_data, dev_data, lr=lr, lr_step_size=int(lr_step_size), lr_gamma=lr_gamma,
            batch_size=int(batch_size), eval_batch_size=int(eval_batch_size), eval_interval=int(eval_interval),
            rollout_steps=int(rollout_steps), time_step_size=tss, rollout_grad_steps=grad_steps,
            input_noise_std=float(input_noise_std), noise_seed=int(noise_seed), noise_every_step=noise_every_step,
            dev_rollout_steps=dev_rollout_steps, dev_time_step_size=dev_tss, max_grad_norm=max_grad_norm,
            ema_decay=ema_decay, generator=generator is not None)
        if random_unroll:   # recorded only when set: a fixed-prefix run's record is that of earlier versions
            config.update(random_unroll=True, unroll_seed=int(unroll_seed))
        if teacher_forcing is not None:   # likewise
            config.update(teacher_forcing=_teacher_record(teacher_forcing), teacher_seed=int(teacher_seed))
        state = resume.find_state(output_dir, config)
    model._require_cuda()
    output_dir = Path(output_dir)
    output_dir.mkdir(exist_ok=True, parents=True)

    optimizer = FusedAdam(model.parameters(), lr=lr, max_grad_norm=max_grad_norm, ema_decay=ema_decay)
    scheduler = torch.optim.lr_scheduler.StepLR(optimizer, step_size=lr_step_size, gamma=lr_gamma)
    start_epoch, global_step = 0, 0
    train_losses: List[float] = []
    grad_norms: List[float] = []
    if state is not None:   # before the graphs are captured: they hold raw pointers to the optimizer state
        model.load_state_dict(state["model"])
        optimizer.load_state_dict(state["optimizer"])
        scheduler.load_state_dict(state["scheduler"])
        resume.restore_rng(state, generator)
        start_epoch, global_step = state["epoch"] + 1, state["global_step"]
        train_losses, grad_norms = list(state["train_losses"]), list(state.get("grad_norms", []))
    with torch.cuda.device(dev):
        frames = as_device_frames(train_data, dev)
        dev_frames = None
        if dev_windows is not None:
            dev_frames = as_device_frames(dev_data, dev)
            _check_chain(dev_frames, dev_windows, dev_rollout_steps, dev_tss, what="dev_data")
        n = frames.n
        ema_model = None if ema_decay is None else _ema_shadow(model)
        noise = dict(noise_std=input_noise_std, noise_seed=int(noise_seed))
        if windows is not None:
            _check_chain(frames, windows, rollout_steps, tss)
        graphs = None   # a resumed run with no epoch left to train captures nothing
        if start_epoch < num_epochs:
            if windows is None:
                graphs = _StepGraphs(model, frames, batch_size, optimizer, **noise)
            else:
                graphs = _RolloutStepGraphs(model, frames, batch_size, optimizer, windows.size, rollout_steps,
                                            tss, grad_steps, noise_every_step=noise_every_step,
                                            random_unroll=random_unroll, unroll_seed=int(unroll_seed),
                                            teacher=teacher_probs is not None, teacher_seed=int(teacher_seed), **noise)
        print("====== Training ======")
        print(f"# batch: {batch_size}")
        print(f"# examples: {n}")
        if windows is not None:
            print(f"# rollout steps: {rollout_steps}, windows: {windows.size}")
            if grad_steps < rollout_steps:
                if random_unroll:
                    print(f"# trained steps: {grad_steps} after a random prefix of 0..{rollout_steps - grad_steps} "
                          f"steps (pushforward, unroll seed {int(unroll_seed)})")
                else:
                    print(f"# trained steps: the last {grad_steps} (pushforward)")
        if teacher_probs is not None:
            print(f"# teacher forcing: p = {teacher_probs[0]} .. {teacher_probs[-1]} over the epochs, seed "
                  f"{int(teacher_seed)}")
        if input_noise_std > 0:
            every = ", on every rollout step" if noise_every_step and windows is not None else ""
            print(f"# input noise std: {input_noise_std}, seed {int(noise_seed)}{every}")
        if max_grad_norm is not None:
            print(f"# max grad norm: {max_grad_norm}")
        if ema_decay is not None:
            print(f"# ema decay: {ema_decay} (evaluated and saved: the EMA weights)")
        if dev_windows is not None:
            print(f"# dev rollout steps: {dev_rollout_steps}, windows: {dev_windows.size} (checkpoints scored by rollout "
                  "nmse)")
        print(f"# step: {-(-(n if windows is None else windows.size) // batch_size)}")
        print(f"# epoch: {num_epochs}")
        if state is not None:
            print(f"# resumed from epoch {state['epoch']} (step {global_step}): {output_dir / resume.STATE_NAME}")
        start_time = time.time()
        try:
            for ep in range(start_epoch, num_epochs):
                ep_start_time = time.time()
                lr_ep = optimizer.param_groups[0]["lr"]
                if windows is None:
                    perm = epoch_permutation(n, batch_size, generator)
                else:
                    perm = windows[epoch_permutation(windows.size, batch_size, generator)]
                if teacher_probs is not None:
                    log = graphs.epoch(perm, lr_ep, global_step + 1, teacher_prob=teacher_probs[ep])
                else:
                    log = graphs.epoch(perm, lr_ep, global_step + 1)
                ep_train_losses = [float(v) for v in log[:, 3]]
                if max_grad_norm is not None:
                    grad_norms += [float(v) for v in graphs.norms]
                for step in range(graphs.steps):
                    global_step += 1
                    if global_step % log_interval == 0:
                        line = dict(ep=ep, step=step, mse=f"{float(log[step, 0]):.3e}", nmse=f"{float(log[step, 3]):.3e}",
                                    lr=f"{scheduler.get_last_lr()[0]:.3e}", time=round(time.time() - start_time))
                        if max_grad_norm is not None:
                            line["grad_norm"] = f"{float(graphs.norms[step]):.3e}"
                        print(line)
                with warnings.catch_warnings():   # the optimizer steps ran inside the graph, not through .step()
                    warnings.filterwarnings("ignore", message=r"Detected call of `lr_scheduler\.step\(\)` before")
                    scheduler.step()
                train_losses += ep_train_losses
                if (ep + 1) % eval_interval == 0:
                    dev_eval_draw(generator)
                    ckpt_dir = output_dir / f"ckpt-{ep}"
                    ckpt_dir.mkdir(exist_ok=True, parents=True)
                    if dev_frames is None:
                        dev_frames = as_device_frames(dev_data, dev)
                    eval_model = model
                    if ema_model is not None:   # evaluate and save the EMA weights
                        optimizer.copy_ema_to(ema_model)
                        eval_model = ema_model
                    dev_scores = evaluate_auto(eval_model, dev_frames, batch_size=eval_batch_size)["scores"]
                    dump_json(dev_scores, ckpt_dir / "dev_scores.json")
                    dump_json(ep_train_losses, ckpt_dir / "train_loss.json")
                    ckpt_path = ckpt_dir / "model.pt"
                    print(f"Saving checkpoint to {ckpt_path}")
                    if ckpt_path.exists():
                        ckpt_backup_path = ckpt_dir / "backup_model.pt"
                        print(f"Backing up old checkpoint to {ckpt_backup_path}")
                        copyfile(ckpt_path, ckpt_backup_path)
                    torch.save(eval_model.state_dict(), ckpt_path)
                    dev_loss = np.mean(dev_scores["all"]["nmse"])
                    if dev_windows is None:
                        ep_scores = dict(ep=ep, train_loss=np.mean(ep_train_losses), dev_loss=dev_loss,
                                         time=time.time() - ep_start_time)
                    else:
                        rollout = _evaluate_rollout(eval_model, dev_frames, dev_windows, dev_rollout_steps, dev_tss)
                        dump_json(rollout, ckpt_dir / "dev_rollout_scores.json")
                        ep_scores = dict(ep=ep, train_loss=np.mean(ep_train_losses), dev_loss=rollout["loss"],
                                         dev_loss_single_step=dev_loss, time=time.time() - ep_start_time)
                    dump_json(ep_scores, ckpt_dir / "scores.json")
                if resumable and ((ep + 1) % eval_interval == 0 or ep == num_epochs - 1):   # after the checkpoint
                    resume.write_state(resume.build_state(ep, global_step, model, optimizer, scheduler, generator,
                                                          train_losses, grad_norms if max_grad_norm is not None else None,
                                                          config), output_dir)
        finally:
            del graphs   # the graphs and their static buffers go with the call
    print("====== Training done ======")
    dump_json(train_losses, output_dir / "train_losses.json")
    out = dict(train_losses=train_losses, optimizer=optimizer, start_epoch=start_epoch)
    if max_grad_norm is not None:
        dump_json(grad_norms, output_dir / "grad_norms.json")
        out["grad_norms"] = grad_norms
    if ema_model is not None:
        optimizer.copy_ema_to(ema_model)
        out["ema_model"] = ema_model
    return out
