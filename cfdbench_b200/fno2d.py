"""Drop-in `Fno2d` for CFDBench backed by the sm_90a kernels in libcfdbench_b200.so.

Mirrors the reference module's public surface (reference src/models/fno/fno2d.py:115-295):
same constructor keywords as `utils/autoregressive.py:114-125` passes, same parameter names /
shapes / dtypes in `state_dict()` (SURVEY.md 8b: fc0, blocks.{l}.conv0.weights1|weights2 (complex64),
blocks.{l}.w0, fc1, fc2), same `forward / generate / generate_many` semantics, same return types.
The sub-modules below are *parameter holders only*: all arithmetic happens in the CUDA library
(`cfdbench_b200._lib`), there is no PyTorch/CPU fallback path.

Extras that the reference does not have (all optional, defaults keep reference behaviour):
  * `act_dtype="bfloat16"`: hidden activations are stored as bf16 between kernels (fp32 arithmetic).
  * `generate_many(..)` runs the whole rollout in one native call; host tensors in -> host tensors out
    through `fno_rollout_host` (H2D + rollout + D2H on one stream).
  * `enable_data_parallel()`: all-reduce of one flat gradient buffer (NCCL) inside backward.
  * `rollout(..)`: a K-step rollout as one differentiable call whose backward recomputes each step, so its memory
    grows by frames, not by saved activations, with K.
Frames: 64x64 runs the 64x64 kernels (either storage mode); any other H x W with 24 <= H, W <= 128 (CFDBench's tube
and dam problems: 66x65) runs the grid-generic fp32 kernels (fno_grid_* in the C ABI), routed by `inputs.shape[-2:]`.
Like the reference, `forward` / `generate` are differentiable w.r.t. `inputs` and `case_params` (not `mask`), also with
every parameter frozen.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Dict, List, NamedTuple, Optional

import numpy as np
import torch
import torch.nn as nn
from torch import Tensor

from . import _lib
from .base_model import AutoCfdModel
from .data import check_rollout_noise, check_teacher_forcing

H = W = 64
HIDDEN = 32
MODES = 12
NMODES = 2 * MODES * MODES  # 288
PROJ = 128
# A host-tensor single step of a large batch is cut into this many equal batch chunks, so that one chunk's copies overlap
# another's kernels.  More chunks run the kernels at batch sizes where their fixed per-launch costs dominate.
HOST_CHUNKS = 2


class SpectralConv2d_fast(nn.Module):
    """Parameter holder for the Fourier weights; init as reference fno2d.py:30-51
    (scale * torch.rand(cfloat), scale = 1/(Cin*Cout))."""

    def __init__(self, in_channels: int, out_channels: int, modes1: int, modes2: int, device=None):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.modes1, self.modes2 = modes1, modes2
        self.scale = 1 / (in_channels * out_channels)
        # generated on CPU then moved so that the RNG stream matches the reference's initialisation order
        self.weights1 = nn.Parameter(
            (self.scale * torch.rand(in_channels, out_channels, modes1, modes2, dtype=torch.cfloat)).to(device))
        self.weights2 = nn.Parameter(
            (self.scale * torch.rand(in_channels, out_channels, modes1, modes2, dtype=torch.cfloat)).to(device))

    def forward(self, x):  # pragma: no cover
        raise RuntimeError("SpectralConv2d_fast is a parameter holder; call Fno2d.forward")


class FnoBlock(nn.Module):
    """Parameter holder: conv0 (spectral weights) + w0 (1x1 conv), reference fno2d.py:85-104."""

    def __init__(self, in_chan: int, out_chan: int, modes1: int, modes2: int, device=None):
        super().__init__()
        self.conv0 = SpectralConv2d_fast(in_chan, out_chan, modes1, modes2, device=device)
        self.w0 = nn.Conv2d(in_chan, out_chan, 1).to(device)

    def forward(self, x):  # pragma: no cover
        raise RuntimeError("FnoBlock is a parameter holder; call Fno2d.forward")


def _ptr(t: Optional[Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def capture_graph(run) -> torch.cuda.CUDAGraph:
    """A CUDA graph of the launches `run()` issues on the current stream.  capture_begin / capture_end directly: the
    torch.cuda.graph() context manager also runs gc.collect() and empty_cache(), which turns the caller's next
    allocation into a multi-millisecond cudaMalloc.  Nothing is allocated during a capture (all buffers are static), so
    no private pool is needed."""
    graph = torch.cuda.CUDAGraph()
    graph.capture_begin(capture_error_mode="thread_local")
    try:
        run()
    finally:
        graph.capture_end()
    return graph


@contextlib.contextmanager
def side_stream(device):
    """Run the block (warm-ups and captures) on a new stream that starts after the current stream's work; the current
    stream then waits for it."""
    cur = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device=device)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        yield
    cur.wait_stream(side)


class _Route(NamedTuple):
    """The kernels that run (gh, gw) frames (`Fno2d._route`): the 64x64 kernels (fno_X, either storage mode) or the
    grid-generic fp32 kernels (fno_grid_X).  The two take the same arguments in the same order except the tail: (batch,
    act_dtype, stream) for 64x64, (batch, h, w, stream) for grids."""
    gh: int
    gw: int
    grid: bool
    act: int   # ACT_F32 on the grid route

    @property
    def act_dtype(self) -> torch.dtype:
        return torch.bfloat16 if self.act == _lib.ACT_BF16 else torch.float32

    def call(self, name: str, *args) -> None:
        """fno_<name> or fno_grid_<name> on `args`: the shared arguments, then batch and stream.  "backward" is
        fno_backward_inputs on 64x64 (with null d_inputs and d_case_params it issues exactly fno_backward's launches)."""
        lib = _lib.load()
        *head, stream = args
        if self.grid:
            fn = "fno_grid_" + name
            status = getattr(lib, fn)(*head, self.gh, self.gw, stream)
        else:
            fn = "fno_backward_inputs" if name == "backward" else "fno_" + name
            status = getattr(lib, fn)(*head, self.act, stream)
        _lib.check(status, fn)

    def bwd_partials_bytes(self) -> int:
        lib = _lib.load()
        return lib.fno_grid_bwd_partials_bytes(self.gh, self.gw) if self.grid else lib.fno_bwd_partials_bytes()


def _refuse_mask_grad(mask: Tensor) -> None:
    if mask.requires_grad:
        # the masked projection keeps no unmasked output, so dL/dmask cannot be formed -- say so instead of silently
        # returning None
        raise NotImplementedError("cfdbench_b200.Fno2d: gradients w.r.t. the mask are not implemented (inputs, "
                                  "case_params and parameters are differentiable)")


class _TrainFn(torch.autograd.Function):
    """One autograd node for the whole network: forward = fno_forward_train, backward = fno_backward_inputs (parameter
    gradients and / or the gradients w.r.t. inputs / case_params).  Every call keeps its own saved activations, so
    forward k+1 may run before backward k (unrolled training through rollouts)."""

    @staticmethod
    def forward(ctx, model: "Fno2d", inputs: Tensor, mask: Tensor, case_params: Tensor, *params: Tensor):
        _refuse_mask_grad(mask)
        preds, saved = model._native_forward_train(inputs, mask, case_params)
        ctx.model = model
        ctx.saved_native = saved
        ctx.save_for_backward(inputs, mask, case_params)
        return preds

    @staticmethod
    def backward(ctx, dpreds: Tensor):
        inputs, mask, case_params = ctx.saved_tensors
        model: "Fno2d" = ctx.model
        if ctx.saved_native is None:
            raise RuntimeError("cfdbench_b200.Fno2d: backward through the same forward a second time (the saved native "
                               "activations were released after the first backward; run forward again)")
        need = ctx.needs_input_grad   # (model, inputs, mask, case_params, *params)
        d_inputs = torch.empty_like(inputs) if need[1] else None
        d_cp = torch.empty_like(case_params) if need[3] else None
        grads = model._native_backward(inputs, mask, case_params, _lib.aligned(dpreds.float()), ctx.saved_native,
                                       any(need[4:]), d_inputs, d_cp)
        ctx.saved_native = None   # the saved activations (up to 1.2 GB at B=256) are released with the first backward
        if grads is None:
            grads = [None] * (len(need) - 4)
        return (None, d_inputs, None, d_cp, *grads)


class _RolloutFn(torch.autograd.Function):
    """One autograd node for a whole K-step rollout (backpropagation through time).  Forward = the native rollout
    training forward: K training forwards into ONE reused saved set, keeping only the K predicted frames.  Backward = one
    native sweep, s = K-1 .. 0, that recomputes step s's saved set from its stored input frame and runs step s's backward
    with the upstream gradient dpreds_s + carry (carry = dL/d(frame fed to step s+1)), accumulating the parameter and
    case-parameter gradients.  Memory: the K+1 frames and one saved set instead of K saved sets.  With `noise` (a
    RolloutNoise) or `teacher` (a TeacherForcing) the frames the steps were fed are kept as well, one more frame per
    step, and the sweep recomputes from them; with `teacher` it also keeps the flags, which gate the hand-off."""

    @staticmethod
    def forward(ctx, model: "Fno2d", inputs: Tensor, mask: Tensor, case_params: Tensor, steps: int, noise, teacher,
                *params: Tensor):
        _refuse_mask_grad(mask)
        seq, fed = model._native_rollout_train(inputs, mask, case_params, steps, noise, teacher)
        ctx.model, ctx.steps, ctx.noise = model, steps, noise
        ctx.save_for_backward(inputs, mask, case_params, seq, fed, None if teacher is None else teacher.flags)
        return seq

    @staticmethod
    def backward(ctx, dseq: Tensor):
        inputs, mask, case_params, seq, fed, flags = ctx.saved_tensors
        model: "Fno2d" = ctx.model
        need = ctx.needs_input_grad   # (model, inputs, mask, case_params, steps, noise, teacher, *params)
        d_inputs = torch.empty_like(inputs) if need[1] else None
        d_cp = torch.empty_like(case_params) if need[3] else None
        grads = model._native_rollout_backward(inputs, mask, case_params, seq, _lib.aligned(dseq.float()), ctx.steps,
                                               any(need[7:]), d_inputs, d_cp, ctx.noise, fed, flags)
        if grads is None:
            grads = [None] * (len(need) - 7)
        return (None, d_inputs, None, d_cp, None, None, None, *grads)


class Fno2d(AutoCfdModel):
    def __init__(
        self,
        in_chan: int,
        out_chan: int,
        n_case_params: int,
        loss_fn: nn.Module,
        num_layers: int,
        modes1: int = 12,
        modes2: int = 12,
        hidden_dim: int = 20,
        padding: Optional[int] = None,
        act_dtype: str = "float32",
        device=None,
    ):
        super().__init__(loss_fn)
        if (hidden_dim, modes1, modes2) != (HIDDEN, MODES, MODES):
            raise ValueError(
                f"cfdbench_b200.Fno2d is specialised on hidden_dim=32, modes=12x12 (CFDBench's FNO config, "
                f"reference src/args.py:187-197); got hidden_dim={hidden_dim}, modes=({modes1},{modes2})")
        if in_chan != 2 or out_chan != 2:
            raise ValueError("cfdbench_b200.Fno2d supports in_chan=out_chan=2 ((u,v) fields) only")
        if padding is not None:
            raise ValueError("padding is not supported (reference init_model never passes it)")
        if not (1 <= num_layers <= _lib.FNO_MAX_LAYERS):
            raise ValueError(f"num_layers must be in 1..{_lib.FNO_MAX_LAYERS}")
        if not (0 <= n_case_params <= 16):
            raise ValueError("n_case_params must be in 0..16")
        if act_dtype not in ("float32", "bfloat16"):
            raise ValueError("act_dtype must be 'float32' or 'bfloat16'")
        self.in_chan, self.out_chan = in_chan, out_chan
        self.n_case_params = n_case_params
        self.num_layers = num_layers
        self.modes1, self.modes2 = modes1, modes2
        self.hidden_dim = hidden_dim
        self.padding = padding
        self.act_dtype = act_dtype
        if device is None:
            # no CPU path: parameters live on the current CUDA device when there is one (this also fixes the
            # reference's missing .cuda() for fno, SURVEY.md 3.1 defect 2).  Without a GPU the module can still be
            # built (state_dict round trips, CPU tests of the host logic) but forward raises.
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        device = torch.device(device)

        # same construction order as the reference so that the RNG stream gives the same initial weights:
        # fc0 -> per block (weights1, weights2, w0) -> fc1 -> fc2   (reference fno2d.py:150-176)
        self.fc0 = nn.Conv2d(in_chan + 1 + 2 + n_case_params, hidden_dim, 1, 1, 0).to(device)
        self.blocks = nn.Sequential(*[FnoBlock(hidden_dim, hidden_dim, modes1, modes2, device=device)
                                      for _ in range(num_layers)])
        self.fc1 = nn.Conv2d(hidden_dim, PROJ, 1, 1, 0).to(device)
        self.fc2 = nn.Conv2d(PROJ, out_chan, 1, 1, 0).to(device)

        self._pack_key = None
        self._packed: dict = {}
        self._ws_cache: dict = {}
        self._dp_group = None
        self._dp_enabled = False
        # CUDA-graph replay of device-resident rollouts: one capture per (batch, steps), the 18 launches of every
        # step replayed as one graph (B=256: 591 -> 544 us/step, B=1: 2.09 -> 1.48 ms per 20 steps).  False = launch
        # every kernel on the stream.
        self.graph_rollout = True
        self.fused_block = True  # bf16 storage, inference: inv_kx + block_tc replaced by block_fused_kernel
        self.max_graphs = 8
        self._graphs: dict = {}
        # True: 64x64 frames in float32 storage also run the grid-generic kernels (fno_grid_*), which cross-checks the two
        # paths; False (default): 64x64 frames run the 64x64 kernels
        self.generic_grid_at_64 = False
        # graphs of `rollout`'s training forward and backward sweep, one capture per (batch, steps, grid, storage[, which
        # gradients]).  They read graph-owned copies of the packed weights, refreshed before a replay when the weights
        # changed, so they survive optimizer steps (the graphs above are dropped when the weights change).
        self._train_graphs: dict = {}

    # ------------------------------------------------------------------------------------ plumbing
    def invalidate_packed(self) -> None:
        """Forget the kernel-layout weight images, captured graphs and workspaces.  Called automatically when parameters
        change through the tracked paths (optimizer steps / in-place ops bump `_version`; `.to()` / `.cuda()` / `load_state_dict`
        go through the hooks below).  Writes through `p.data` or raw pointers bump no version counter: call this by hand
        after such writes (EMA swaps, manual weight edits)."""
        self._pack_key = None
        self._packed = {}
        self._graphs = {}
        self._ws_cache = {}
        self._train_graphs = {}

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        if hasattr(self, "_pack_key"):
            self.invalidate_packed()
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self.invalidate_packed()
        return out

    @property
    def device(self) -> torch.device:
        return self.fc0.weight.device

    def _act_code(self) -> int:
        return _lib.ACT_BF16 if self.act_dtype == "bfloat16" else _lib.ACT_F32

    def _require_cuda(self):
        if self.device.type != "cuda":
            raise _lib.FnoNativeError(
                "cfdbench_b200.Fno2d has no CPU path: parameters are on %s; move the model to a CUDA device" % self.device)

    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _needs_grad(self, *tensors: Tensor) -> bool:
        """Whether a call on `tensors` has to build an autograd graph."""
        return torch.is_grad_enabled() and (any(t.requires_grad for t in tensors)
                                            or any(p.requires_grad for p in self.parameters()))

    def _pack(self, need_bwd: bool = False) -> dict:
        """(Re)build kernel-layout weights when any parameter changed (version counters / pointers)."""
        plist = list(self.parameters())
        key = (str(self.device),) + tuple((p.data_ptr(), p._version) for p in plist)
        pk = self._packed
        if key != self._pack_key:
            lib = _lib.load()
            dev = self.device
            for p in plist:
                if not p.is_contiguous():
                    raise _lib.FnoNativeError("parameters must be contiguous")
            pk = {"wk": [], "w0t": [], "wkT": None}
            st = self._stream()
            for blk in self.blocks:
                pk["wk"].append(self._mix_operand(blk, 0))
                pk["w0t"].append(blk.w0.weight.detach().view(HIDDEN, HIDDEN).t().contiguous())
            if "gx" not in self._packed or self._packed["gx"].device != dev:
                lin = torch.tensor(np.linspace(0, 1, H), dtype=torch.float)  # as reference fno2d.py:250-252
                pk["gx"] = lin.to(dev)
                pk["gy"] = lin.clone().to(dev)
            else:
                pk["gx"], pk["gy"] = self._packed["gx"], self._packed["gy"]
            w = _lib.FnoWeights()
            w.n_layers, w.n_case_params = self.num_layers, self.n_case_params
            w.fc0_w, w.fc0_b = self.fc0.weight.data_ptr(), self.fc0.bias.data_ptr()
            for l, blk in enumerate(self.blocks):
                w.spec_wk[l] = pk["wk"][l].data_ptr()
                w.w0t[l] = pk["w0t"][l].data_ptr()
                w.w0_b[l] = blk.w0.bias.data_ptr()
            w.fc1_w, w.fc1_b = self.fc1.weight.data_ptr(), self.fc1.bias.data_ptr()
            w.fc2_w, w.fc2_b = self.fc2.weight.data_ptr(), self.fc2.bias.data_ptr()
            w.gx, w.gy = pk["gx"].data_ptr(), pk["gy"].data_ptr()
            pk["struct"] = w
            pk["coords"] = {(H, W): (w, pk["gx"], pk["gy"])}   # (gh, gw) -> (struct, gx, gy), see _coords
            self._packed, self._pack_key = pk, key
            self._graphs.clear()
        if need_bwd and pk.get("wkT") is None:
            lib = _lib.load()
            st = self._stream()
            pk["wkT"] = []
            wb = _lib.FnoWeightsBwd()
            for l, blk in enumerate(self.blocks):
                wkT = self._mix_operand(blk, 1)
                pk["wkT"].append(wkT)
                wb.spec_wkT[l] = wkT.data_ptr()
                wb.w0[l] = blk.w0.weight.data_ptr()
            pk["struct_bwd"] = wb
        return pk

    def _mix_operand(self, blk: "FnoBlock", conj_transpose: int) -> Tensor:
        """weights1/2 -> the tensor-core operand image fno_mode_mix consumes (one launch)."""
        lib = _lib.load()
        wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device=self.device)
        _lib.check(lib.fno_pack_mix_operand_from_weights(blk.conv0.weights1.data_ptr(), blk.conv0.weights2.data_ptr(),
                                                         wop.data_ptr(), conj_transpose, self._stream()),
                   "fno_pack_mix_operand_from_weights")
        return wop

    def _workspace(self, batch: int, route: Optional[_Route] = None, slot: int = 0):
        """(FnoWorkspace, bufs) for `batch` samples on the kernels of `route` (default: the 64x64 kernels, whatever
        generic_grid_at_64 says); `slot` keeps apart 64x64 workspaces of one batch size that are in use together."""
        route = route or _Route(H, W, False, self._act_code())
        gh, gw = route.gh, route.gw
        key = ("grid", batch, gh, gw, self.device) if route.grid else (batch, self.act_dtype, self.device, slot,
                                                                        self.fused_block)
        ws = self._ws_cache.get(key)
        if ws is None:
            dev = self.device
            adt = route.act_dtype
            bufs = dict(
                act0=torch.empty(batch, HIDDEN, gh, gw, dtype=adt, device=dev),
                act1=torch.empty(batch, HIDDEN, gh, gw, dtype=adt, device=dev),
                xm=torch.empty(NMODES, batch, HIDDEN, dtype=torch.complex64, device=dev),
                ym=torch.empty(NMODES, batch, HIDDEN, dtype=torch.complex64, device=dev),
                z=torch.empty(batch, gh, 2 * MODES, HIDDEN, dtype=torch.float32, device=dev),
            )
            st = _lib.FnoWorkspace()
            st.act[0], st.act[1] = bufs["act0"].data_ptr(), bufs["act1"].data_ptr()
            st.xm, st.ym, st.z = bufs["xm"].data_ptr(), bufs["ym"].data_ptr(), bufs["z"].data_ptr()
            if route.act == _lib.ACT_BF16 and self.fused_block:
                # operand image of the fused output stage (fno_block_fused): inference never touches ym / z then
                bufs["ym_img"] = torch.empty(_lib.load().fno_ym_image_bytes(batch), dtype=torch.uint8, device=dev)
                st.ym_img = bufs["ym_img"].data_ptr()
            ws = (st, bufs)
            if len(self._ws_cache) > 16:
                self._ws_cache.clear()
            self._ws_cache[key] = ws
        return ws

    def _route(self, gh: int, gw: int) -> _Route:
        """The kernels that run (gh, gw) frames: 64x64 runs the 64x64 kernels in either storage mode (the grid-generic
        kernels with generic_grid_at_64, which cross-checks the two), any other grid with 24 <= H, W <= 128 the
        grid-generic fp32 kernels.  Raises ValueError for any other grid or a storage mode its kernels do not run."""
        gh, gw = int(gh), int(gw)
        if (gh, gw) == (H, W):
            if not self.generic_grid_at_64:
                return _Route(gh, gw, False, self._act_code())
            if self.act_dtype != "float32":
                raise ValueError("generic_grid_at_64 needs act_dtype='float32'")
        else:
            if not (_lib.GRID_MIN <= gh <= _lib.GRID_MAX and _lib.GRID_MIN <= gw <= _lib.GRID_MAX):
                raise ValueError(f"cfdbench_b200.Fno2d supports {H}x{W} frames and grids with {_lib.GRID_MIN} <= H, "
                                 f"W <= {_lib.GRID_MAX}; got {gh}x{gw}")
            if self.act_dtype != "float32":
                raise ValueError(f"cfdbench_b200.Fno2d: act_dtype={self.act_dtype!r} is supported on {H}x{W} frames "
                                 f"only; the {gh}x{gw} grid runs with act_dtype='float32'")
        return _Route(gh, gw, True, _lib.ACT_F32)

    def _prep_inputs(self, inputs: Tensor, case_params: Tensor, mask: Optional[Tensor]):
        """Inputs, case parameters and the (B, 1, H, W) mask as contiguous, 16-byte aligned float32 device tensors
        (`_lib.aligned`: a view that starts inside its storage is copied); the mask follows the input's grid, which
        `_route` checks."""
        if inputs.dim() != 4 or inputs.shape[1] != self.in_chan:
            raise ValueError(f"inputs must be (B,{self.in_chan},H,W); got {tuple(inputs.shape)}")
        gh, gw = self._route(*inputs.shape[-2:])[:2]
        b = inputs.shape[0]
        dev = self.device
        inputs = _lib.aligned(inputs.to(device=dev, dtype=torch.float32, non_blocking=True))
        if case_params.shape != (b, self.n_case_params):
            raise ValueError(f"case_params must be ({b},{self.n_case_params}); got {tuple(case_params.shape)}")
        case_params = case_params.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
        if mask is None:
            mask4 = torch.ones((b, 1, gh, gw), device=dev)  # reference fno2d.py:197-199
        else:
            mask4 = mask.unsqueeze(1) if mask.dim() == 3 else mask
            if tuple(mask4.shape) != (b, 1, gh, gw):
                raise ValueError(f"mask must be (B,{gh},{gw}) or (B,1,{gh},{gw}); got {tuple(mask.shape)}")
            mask4 = _lib.aligned(mask4.to(device=dev, dtype=torch.float32, non_blocking=True))
        return inputs, case_params, mask4

    def _coords(self, pk: dict, gh: int, gw: int) -> tuple:
        """(weight struct, gx, gy) of (gh, gw) frames: the packed weight struct with coordinate tables
        float32(np.linspace(0, 1, n)) of the frame's size; on 64x64 pk["struct"] and its own tables."""
        ent = pk["coords"].get((gh, gw))
        if ent is None:
            gx = torch.tensor(np.linspace(0, 1, gh), dtype=torch.float).to(self.device)
            gy = torch.tensor(np.linspace(0, 1, gw), dtype=torch.float).to(self.device)
            st = _lib.FnoWeights.from_buffer_copy(pk["struct"])
            st.gx, st.gy = gx.data_ptr(), gy.data_ptr()
            ent = pk["coords"][(gh, gw)] = (st, gx, gy)
        return ent

    def _saved_set(self, b: int, route: _Route) -> tuple:
        """The saved activations of one training forward of `b` samples: (FnoTrainSaved, acts, pres, xms)."""
        dev, L, gh, gw = self.device, self.num_layers, route.gh, route.gw
        acts = [torch.empty(b, HIDDEN, gh, gw, dtype=route.act_dtype, device=dev) for _ in range(L + 1)]
        pres = [torch.empty(b, HIDDEN, gh, gw, dtype=torch.float32, device=dev) for _ in range(L)]
        xms = [torch.empty(NMODES, b, HIDDEN, dtype=torch.complex64, device=dev) for _ in range(L)]
        sv = _lib.FnoTrainSaved()
        for l in range(L + 1):
            sv.act[l] = acts[l].data_ptr()
        for l in range(L):
            sv.pre[l], sv.xm[l] = pres[l].data_ptr(), xms[l].data_ptr()
        return sv, acts, pres, xms

    def _bwd_scratch(self, b: int, route: _Route) -> tuple:
        """The backward's scratch for `b` samples: (FnoBwdScratch, bufs = two d buffers, dz1, gm, gwk, partials)."""
        dev, gh, gw = self.device, route.gh, route.gw
        bufs = dict(
            d0=torch.empty(b, HIDDEN, gh, gw, dtype=torch.float32, device=dev),
            d1=torch.empty(b, HIDDEN, gh, gw, dtype=torch.float32, device=dev),
            dz1=torch.empty(min(b, _lib.BWD_CHUNK), PROJ, gh, gw, dtype=torch.float32, device=dev),
            gm=torch.empty(NMODES, b, HIDDEN, dtype=torch.complex64, device=dev),
            gwk=torch.empty(NMODES, HIDDEN, HIDDEN, dtype=torch.complex64, device=dev),
            partials=torch.empty(route.bwd_partials_bytes(), dtype=torch.uint8, device=dev),
        )
        sc = _lib.FnoBwdScratch()
        sc.d[0], sc.d[1] = bufs["d0"].data_ptr(), bufs["d1"].data_ptr()
        sc.dz1, sc.gm, sc.gwk = bufs["dz1"].data_ptr(), bufs["gm"].data_ptr(), bufs["gwk"].data_ptr()
        sc.partials = bufs["partials"].data_ptr()
        return sc, bufs

    # ------------------------------------------------------------------------------ native calls
    def _native_forward(self, inputs: Tensor, mask4: Tensor, case_params: Tensor) -> Tensor:
        b = inputs.shape[0]
        pk = self._pack()
        route = self._route(*inputs.shape[-2:])
        ws, _ = self._workspace(b, route)
        preds = torch.empty(b, self.out_chan, route.gh, route.gw, dtype=torch.float32, device=self.device)
        route.call("forward", C.byref(self._coords(pk, route.gh, route.gw)[0]), inputs.data_ptr(), mask4.data_ptr(),
                   case_params.data_ptr(), preds.data_ptr(), C.byref(ws), b, self._stream())
        return preds

    def _native_forward_train(self, inputs: Tensor, mask4: Tensor, case_params: Tensor):
        b = inputs.shape[0]
        pk = self._pack(need_bwd=True)
        route = self._route(*inputs.shape[-2:])
        ws, _ = self._workspace(b, route)
        saved = self._saved_set(b, route)
        preds = torch.empty(b, self.out_chan, route.gh, route.gw, dtype=torch.float32, device=self.device)
        route.call("forward_train", C.byref(self._coords(pk, route.gh, route.gw)[0]), inputs.data_ptr(),
                   mask4.data_ptr(), case_params.data_ptr(), preds.data_ptr(), C.byref(saved[0]), C.byref(ws), b,
                   self._stream())
        return preds, saved

    def _grad_layout(self):
        """(name, param, offset, n_real) for one flat float32 gradient buffer, parameter order."""
        out, off = [], 0
        for name, p in self.named_parameters():
            n = p.numel() * (2 if p.is_complex() else 1)
            out.append((name, p, off, n))
            off += n
        return out, off

    def _grad_buffers(self):
        """One flat float32 gradient buffer, its per-parameter views (parameter order) and the FnoGrads struct."""
        layout, total = self._grad_layout()
        flat = torch.empty(total, dtype=torch.float32, device=self.device)
        views: Dict[str, Tensor] = {}
        for name, p, off, n in layout:
            seg = flat[off:off + n]
            views[name] = torch.view_as_complex(seg.view(*p.shape, 2)) if p.is_complex() else seg.view(p.shape)
        g = _lib.FnoGrads()
        g.fc0_w, g.fc0_b = views["fc0.weight"].data_ptr(), views["fc0.bias"].data_ptr()
        for l in range(self.num_layers):
            g.spec_w1[l] = views[f"blocks.{l}.conv0.weights1"].data_ptr()
            g.spec_w2[l] = views[f"blocks.{l}.conv0.weights2"].data_ptr()
            g.w0_w[l] = views[f"blocks.{l}.w0.weight"].data_ptr()
            g.w0_b[l] = views[f"blocks.{l}.w0.bias"].data_ptr()
        g.fc1_w, g.fc1_b = views["fc1.weight"].data_ptr(), views["fc1.bias"].data_ptr()
        g.fc2_w, g.fc2_b = views["fc2.weight"].data_ptr(), views["fc2.bias"].data_ptr()
        return flat, views, g

    def _native_backward(self, inputs, mask4, case_params, dpreds, saved_native, want_params: bool = True,
                         d_inputs: Optional[Tensor] = None, d_cp: Optional[Tensor] = None):
        """Parameter gradients in parameter order (None when `want_params` is false), from one native call:
        fno_backward_inputs on 64x64 frames (with `d_inputs` and `d_cp` None it issues exactly fno_backward's launches),
        fno_grid_backward on other grids.  It also writes dL/dinputs into `d_inputs` and dL/dcase_params into `d_cp` when
        given.  Those are per sample: with data parallel enabled only the parameter gradients are all-reduced."""
        if self.n_case_params == 0:
            d_cp = None   # a (B, 0) gradient: nothing to write
        if not want_params and d_inputs is None and d_cp is None:
            return None
        b = inputs.shape[0]
        pk = self._pack(need_bwd=True)
        route = self._route(*inputs.shape[-2:])
        ws, _ = self._workspace(b, route)
        flat = views = g = None
        if want_params:
            flat, views, g = self._grad_buffers()
        sc, scratch = self._bwd_scratch(b, route)   # `scratch` holds the tensors `sc` points into
        route.call("backward", C.byref(self._coords(pk, route.gh, route.gw)[0]), C.byref(pk["struct_bwd"]),
                   inputs.data_ptr(), mask4.data_ptr(), case_params.data_ptr(), dpreds.data_ptr(),
                   C.byref(saved_native[0]), C.byref(g) if g is not None else None, C.byref(sc), C.byref(ws),
                   _ptr(d_inputs), _ptr(d_cp), b, self._stream())
        if g is None:   # data-only backward: no parameter gradients, nothing to all-reduce
            return None
        return self._grad_result(flat, views)

    def _grad_result(self, flat: Tensor, views: Dict[str, Tensor]) -> List[Tensor]:
        """The parameter gradients in parameter order, after one all-reduce (NCCL: ReduceOp.AVG, no division kernel) of
        the whole flat buffer when data parallel is enabled."""
        if self._dp_enabled:
            from .dp import allreduce_mean_
            allreduce_mean_(flat, self._dp_group)
        return [views[name] for name, _ in self.named_parameters()]

    # ---------------------------------------------------------------- training through a rollout (`rollout`)
    def _rollout_state(self, b: int, route: _Route) -> dict:
        """The buffers `rollout` reuses across steps and calls: one saved set, the backward scratch (two d buffers,
        dz1, gm, gwk, partials) and the carry frame."""
        key = ("rollout_train", b, route.gh, route.gw, route.grid, self.act_dtype, self.device)
        st = self._ws_cache.get(key)
        if st is None:
            st = self._train_state(b, route)
            st["bufs"]["carry"] = torch.empty(b, self.out_chan, route.gh, route.gw, dtype=torch.float32,
                                              device=self.device)
            if len(self._ws_cache) > 16:
                self._ws_cache.clear()
            self._ws_cache[key] = st
        return st

    def _train_state(self, b: int, route: _Route) -> dict:
        """One saved set and the backward scratch of a training step of batch `b` (not cached): dict(sv=FnoTrainSaved,
        sc=FnoBwdScratch, bufs=the scratch tensors, saved=(acts, pres, xms)).  Any batch up to `b` can run on them."""
        sv, acts, pres, xms = self._saved_set(b, route)
        sc, bufs = self._bwd_scratch(b, route)
        return dict(sv=sv, sc=sc, bufs=bufs, saved=(acts, pres, xms))

    def _static_weights(self, pk: dict, gh: int, gw: int) -> dict:
        """Graph-owned copies of the packed weight images (and coordinate tables) with the weight structs pointing at
        them; the parameters themselves are read in place.  `_refresh_static_weights` copies a new packing in."""
        src = self._coords(pk, gh, gw)[0]
        wk = [torch.empty_like(t) for t in pk["wk"]]
        w0t = [torch.empty_like(t) for t in pk["w0t"]]
        wkT = [torch.empty_like(t) for t in pk["wkT"]]
        gx = torch.empty(gh, dtype=torch.float32, device=self.device)
        gy = torch.empty(gw, dtype=torch.float32, device=self.device)
        st = _lib.FnoWeights.from_buffer_copy(src)
        sb = _lib.FnoWeightsBwd.from_buffer_copy(pk["struct_bwd"])
        for l in range(self.num_layers):
            st.spec_wk[l], st.w0t[l], sb.spec_wkT[l] = wk[l].data_ptr(), w0t[l].data_ptr(), wkT[l].data_ptr()
        st.gx, st.gy = gx.data_ptr(), gy.data_ptr()
        return dict(struct=st, struct_bwd=sb, dst=wk + w0t + wkT + [gx, gy], src=None)

    def _refresh_static_weights(self, sw: dict, pk: dict, gh: int, gw: int) -> None:
        if sw["src"] is pk:
            return
        _, gx, gy = self._coords(pk, gh, gw)
        for d, s in zip(sw["dst"], pk["wk"] + pk["w0t"] + pk["wkT"] + [gx, gy]):
            d.copy_(s)
        sw["src"] = pk

    def _train_graph(self, key, pk: dict, route: _Route, make_io, run, keep) -> dict:
        """The captured graph of `key` (captured on first use): `make_io()` builds its static buffers, `run(sw, io)`
        issues the native call on them.  Recaptured when a parameter's storage moved."""
        ptrs = tuple(p.data_ptr() for p in self.parameters())
        ent = self._train_graphs.get(key)
        if ent is not None and ent["ptrs"] != ptrs:
            del self._train_graphs[key]
            ent = None
        if ent is None:
            sw = self._static_weights(pk, route.gh, route.gw)
            self._refresh_static_weights(sw, pk, route.gh, route.gw)
            io = make_io()
            with side_stream(self.device):
                run(sw, io)   # warm-up outside capture (kernel attributes, constant tables)
                graph = capture_graph(lambda: run(sw, io))
            ent = dict(graph=graph, io=io, sw=sw, ptrs=ptrs, keep=keep)
            while len(self._train_graphs) >= self.max_graphs:   # oldest capture goes first
                self._train_graphs.pop(next(iter(self._train_graphs)))
            self._train_graphs[key] = ent
        self._refresh_static_weights(ent["sw"], pk, route.gh, route.gw)
        return ent

    def _noise_io(self, noise) -> dict:
        """Device copies of a RolloutNoise's sample indices and step, and the fno_noise descriptor pointing at them
        (kept together: the descriptor holds raw pointers).  A captured graph owns one and refills it per call."""
        io = dict(ids=noise.ids.clone(), step=torch.full((1,), noise.step, dtype=torch.int64, device=self.device))
        io["desc"] = _lib.FnoNoise(noise.std, noise.seed, io["ids"].data_ptr(), io["step"].data_ptr(), None, noise.k0)
        return io

    @staticmethod
    def _refill_noise_io(nio: dict, noise) -> None:
        nio["ids"].copy_(noise.ids)
        nio["step"].fill_(noise.step)   # a fill kernel: no host-to-device copy

    @staticmethod
    def _teacher_io(frames: Optional[Tensor], flags: Tensor) -> dict:
        """Graph-owned copies of a teacher's frames (None for the sweep, which reads only the flags) and flags, and the
        fno_teacher descriptor pointing at them."""
        io = dict(frames=None if frames is None else _lib.aligned(frames.clone()), flags=flags.clone())
        io["desc"] = _lib.FnoTeacher(_ptr(io["frames"]), io["flags"].data_ptr())
        return io

    def _native_rollout_train(self, inputs: Tensor, mask4: Tensor, case_params: Tensor, steps: int, noise=None,
                              teacher=None):
        """(preds, fed): preds (steps, B, 2, H, W) from fno_[grid_]rollout_forward_train: the training forward's kernels,
        so the predictions equal those of chained `generate` calls under autograd bit for bit.  fed is None, or with
        `noise` (a RolloutNoise) the (steps, B, 2, H, W) frames the steps were fed (fno_[grid_]rollout_forward_train_noise:
        slot s holds step s's perturbed input when its stream k0 + s is at least 1).  With `teacher` (a TeacherForcing)
        the call is fno_[grid_]rollout_forward_train_feed and slot s >= 1 of fed always holds step s's input."""
        b = inputs.shape[0]
        route = self._route(*inputs.shape[-2:])
        gh, gw = route.gh, route.gw
        pk = self._pack(need_bwd=True)
        ws, ws_bufs = self._workspace(b, route)
        rs = self._rollout_state(b, route)
        seq = torch.empty(steps, b, self.out_chan, gh, gw, dtype=torch.float32, device=self.device)
        fed = None if noise is None and teacher is None else torch.empty_like(seq)

        def call(st, x, mk, cp, out, nio, tio, fd):
            if tio is not None:
                route.call("rollout_forward_train_feed", C.byref(st), x.data_ptr(), mk.data_ptr(), cp.data_ptr(),
                           out.data_ptr(), steps, C.byref(rs["sv"]), C.byref(ws),
                           None if nio is None else C.byref(nio["desc"]), C.byref(tio["desc"]), fd.data_ptr(), b,
                           self._stream())
            elif nio is None:
                route.call("rollout_forward_train", C.byref(st), x.data_ptr(), mk.data_ptr(), cp.data_ptr(),
                           out.data_ptr(), steps, C.byref(rs["sv"]), C.byref(ws), b, self._stream())
            else:
                route.call("rollout_forward_train_noise", C.byref(st), x.data_ptr(), mk.data_ptr(), cp.data_ptr(),
                           out.data_ptr(), steps, C.byref(rs["sv"]), C.byref(ws), C.byref(nio["desc"]), fd.data_ptr(), b,
                           self._stream())
        if not self.graph_rollout:
            tio = None
            if teacher is not None:
                tio = dict(frames=teacher.frames, flags=teacher.flags)
                tio["desc"] = _lib.FnoTeacher(teacher.frames.data_ptr(), teacher.flags.data_ptr())
            call(self._coords(pk, gh, gw)[0], inputs, mask4, case_params, seq,
                 None if noise is None else self._noise_io(noise), tio, fed)
            return seq, fed
        key = ("fwd", b, steps, gh, gw, route.grid, self.act_dtype,
               None if noise is None else (noise.std, noise.seed, noise.k0), teacher is not None)

        def make_io():
            io = dict(x=inputs.clone(), mk=mask4.clone(), cp=case_params.clone(), seq=torch.empty_like(seq),
                      noise=None, teacher=None, fed=None)
            if noise is not None:
                io["noise"] = self._noise_io(noise)
            if teacher is not None:
                io["teacher"] = self._teacher_io(teacher.frames, teacher.flags)
            if fed is not None:
                io["fed"] = torch.empty_like(seq)
            return io
        ent = self._train_graph(
            key, pk, route, make_io,
            lambda sw, io: call(sw["struct"], io["x"], io["mk"], io["cp"], io["seq"], io["noise"], io["teacher"],
                                io["fed"]),
            (ws_bufs, rs))
        io = ent["io"]
        io["x"].copy_(inputs)
        io["mk"].copy_(mask4)
        io["cp"].copy_(case_params)
        if noise is not None:
            self._refill_noise_io(io["noise"], noise)
        if teacher is not None:
            io["teacher"]["frames"].copy_(teacher.frames)
            io["teacher"]["flags"].copy_(teacher.flags)
        ent["graph"].replay()
        seq.copy_(io["seq"])
        if fed is not None:
            fed.copy_(io["fed"])
        return seq, fed

    def _native_rollout_backward(self, inputs, mask4, case_params, seq, dseq, steps: int, want_params: bool,
                                 d_inputs: Optional[Tensor], d_cp: Optional[Tensor], noise=None,
                                 fed: Optional[Tensor] = None, flags: Optional[Tensor] = None):
        """One native sweep (fno_[grid_]rollout_backward): parameter gradients in parameter order (None when
        `want_params` is false), dL/dinputs into `d_inputs` and dL/dcase_params into `d_cp` when given.  With data
        parallel enabled the flat parameter-gradient buffer is all-reduced once.  With `noise` the sweep
        (fno_[grid_]rollout_backward_noise) recomputes each noisy step from its frame in `fed`; with teacher `flags`
        (fno_[grid_]rollout_backward_feed) every step s >= 1 from fed[s], and the flags gate the hand-off."""
        if self.n_case_params == 0:
            d_cp = None
        if not want_params and d_inputs is None and d_cp is None:
            return None
        b = inputs.shape[0]
        route = self._route(*inputs.shape[-2:])
        gh, gw = route.gh, route.gw
        pk = self._pack(need_bwd=True)
        ws, ws_bufs = self._workspace(b, route)
        rs = self._rollout_state(b, route)
        carry = rs["bufs"]["carry"]

        def call(st, sb, x, mk, cp, sq, dsq, g, din, dcp, nio, tio, fd):
            g = C.byref(g) if g is not None else None
            if tio is not None:
                route.call("rollout_backward_feed", C.byref(st), C.byref(sb), x.data_ptr(), mk.data_ptr(),
                           cp.data_ptr(), sq.data_ptr(), dsq.data_ptr(), steps, C.byref(rs["sv"]), g, C.byref(rs["sc"]),
                           C.byref(ws), None if nio is None else C.byref(nio["desc"]), C.byref(tio["desc"]),
                           fd.data_ptr(), carry.data_ptr(), _ptr(din), _ptr(dcp), b, self._stream())
            elif nio is None:
                route.call("rollout_backward", C.byref(st), C.byref(sb), x.data_ptr(), mk.data_ptr(), cp.data_ptr(),
                           sq.data_ptr(), dsq.data_ptr(), steps, C.byref(rs["sv"]), g, C.byref(rs["sc"]), C.byref(ws),
                           carry.data_ptr(), _ptr(din), _ptr(dcp), b, self._stream())
            else:
                route.call("rollout_backward_noise", C.byref(st), C.byref(sb), x.data_ptr(), mk.data_ptr(),
                           cp.data_ptr(), sq.data_ptr(), dsq.data_ptr(), steps, C.byref(rs["sv"]), g, C.byref(rs["sc"]),
                           C.byref(ws), C.byref(nio["desc"]), fd.data_ptr(), carry.data_ptr(), _ptr(din), _ptr(dcp), b,
                           self._stream())
        flat = views = None
        if not self.graph_rollout:
            g = None
            if want_params:
                flat, views, g = self._grad_buffers()
            tio = None
            if flags is not None:
                tio = dict(flags=flags, desc=_lib.FnoTeacher(None, flags.data_ptr()))
            call(self._coords(pk, gh, gw)[0], pk["struct_bwd"], inputs, mask4, case_params, seq, dseq, g, d_inputs,
                 d_cp, None if noise is None else self._noise_io(noise), tio, fed)
        else:
            def make_io():
                io = dict(x=inputs.clone(), mk=mask4.clone(), cp=case_params.clone(), seq=torch.empty_like(seq),
                          dseq=torch.empty_like(dseq), g=None,
                          din=torch.empty_like(d_inputs) if d_inputs is not None else None,
                          dcp=torch.empty_like(d_cp) if d_cp is not None else None, noise=None, teacher=None, fed=None)
                if want_params:
                    io["flat"], _, io["g"] = self._grad_buffers()
                if noise is not None:
                    io["noise"] = self._noise_io(noise)
                if flags is not None:
                    io["teacher"] = self._teacher_io(None, flags)
                if fed is not None:
                    io["fed"] = torch.empty_like(fed)
                return io
            # the sweep draws no noise: of the descriptor it reads only k0 (the other fields, from the capturing call,
            # are checked and never read), so std, seed, step and ids do not key the capture
            key = ("bwd", b, steps, gh, gw, route.grid, self.act_dtype, want_params, d_inputs is not None,
                   d_cp is not None, None if noise is None else noise.k0, flags is not None)
            ent = self._train_graph(
                key, pk, route, make_io,
                lambda sw, io: call(sw["struct"], sw["struct_bwd"], io["x"], io["mk"], io["cp"], io["seq"], io["dseq"],
                                    io["g"], io["din"], io["dcp"], io["noise"], io["teacher"], io["fed"]), (ws_bufs, rs))
            io = ent["io"]
            for k, t in (("x", inputs), ("mk", mask4), ("cp", case_params), ("seq", seq), ("dseq", dseq)):
                io[k].copy_(t)
            if fed is not None:
                io["fed"].copy_(fed)
            if flags is not None:
                io["teacher"]["flags"].copy_(flags)
            ent["graph"].replay()
            if d_inputs is not None:
                d_inputs.copy_(io["din"])
            if d_cp is not None:
                d_cp.copy_(io["dcp"])
            if want_params:   # the caller owns its gradients: a fresh buffer, never a view of the graph's
                flat, views, _ = self._grad_buffers()
                flat.copy_(io["flat"])
        if not want_params:
            return None
        return self._grad_result(flat, views)   # one all-reduce per backward, not one per step

    # -------------------------------------------------------------------------------- public API
    def enable_data_parallel(self, group=None) -> None:
        """Average gradients over `group` with one all-reduce of the flat gradient buffer at the end of
        backward (the reference has no distributed code; train_auto.py builds no DDP wrapper, so the hook
        lives in the module).  Replicas must start from identical weights."""
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self._dp_group, self._dp_enabled = group, True

    def forward(self, inputs: Tensor, case_params: Tensor, mask: Optional[Tensor] = None,
                label: Optional[Tensor] = None) -> Dict:
        """Same contract as reference fno2d.py:178-242: returns {"preds": (B,2,H,W) float32 masked}
        plus {"loss": dict} when `label` is given.  With grad mode on, `preds` is differentiable w.r.t. the parameters,
        `inputs` and `case_params` (whichever require grad; `mask` does not take gradients), so a frozen model still
        gives d(preds)/d(inputs) and `generate` can be chained for unrolled training."""
        self._require_cuda()
        inputs, case_params, mask4 = self._prep_inputs(inputs, case_params, mask)
        with torch.cuda.device(self.device):
            if self._needs_grad(inputs, case_params, mask4):
                preds = _TrainFn.apply(self, inputs, mask4, case_params, *self.parameters())
            else:
                preds = self._native_forward(inputs, mask4, case_params)
        if label is not None:
            label = label.to(device=self.device, dtype=torch.float32) * mask4
            return dict(preds=preds, loss=self.loss_fn(preds=preds, labels=label))
        return dict(preds=preds)

    def generate(self, inputs: Tensor, case_params: Tensor, mask: Optional[Tensor] = None) -> Tensor:
        return self.forward(inputs=inputs, case_params=case_params, mask=mask)["preds"]

    def generate_many(self, inputs: Tensor, case_params: Tensor, mask: Tensor, steps: int) -> List[Tensor]:
        """reference fno2d.py:269-295.  Returns a list of `steps` tensors (B,c,h,w); tensors live where
        `inputs` lives (host tensors take the H2D -> rollout -> D2H path in one native call).  Always runs without
        autograd (the graph-replayed inference rollout); to train through a rollout, chain `generate` calls."""
        self._require_cuda()
        assert len(inputs.shape) == len(case_params.shape) + 2
        if inputs.dim() == 3:
            inputs, case_params, mask = inputs.unsqueeze(0), case_params.unsqueeze(0), mask.unsqueeze(0)
        assert inputs.shape[0] == case_params.shape[0] == mask.shape[0]
        if steps <= 0:
            return []
        host = inputs.device.type == "cpu"
        with torch.no_grad(), torch.cuda.device(self.device):
            if host:
                seq = self._rollout_host(inputs, case_params, mask, steps)
            else:
                inputs, case_params, mask4 = self._prep_inputs(inputs, case_params, mask)
                seq = self._rollout_device(inputs, case_params, mask4, steps)
        return [seq[s] for s in range(steps)]

    def rollout(self, inputs: Tensor, case_params: Tensor, mask: Optional[Tensor], steps: int, noise=None,
                teacher=None) -> Tensor:
        """`steps` autoregressive steps as one (steps, B, 2, H, W) float32 tensor, trainable through the whole rollout.
        Arguments as `generate_many` ((c,h,w) / (p,) / (h,w) inputs get a batch axis); every grid and storage mode of
        `forward`.  Step s is fed the (masked) prediction of step s-1, computed with the training forward's kernels, so
        the predictions equal those of `steps` chained `generate` calls under autograd bit for bit.

        With autograd on, the result is differentiable w.r.t. the parameters, `inputs` and `case_params` (a `mask` that
        requires grad raises NotImplementedError, as in `forward`).  Unlike chained `generate` calls, each of which keeps
        its own saved activations until backward (about 1 GB per step at B = 256), it keeps only the predicted frames and
        one reused set of saved activations: the backward recomputes each step's activations from its input frame (one
        extra training forward per step) while it sweeps the steps from last to first.  With autograd off it returns the
        same predictions and builds no graph.

        noise = RolloutNoise(std, seed, step, ids, k0) perturbs the frame every step is fed: step s is fed
        `add_input_noise(x_s, mask, ids, std, seed, step, stream=k0 + s)` where x_s is `inputs` (s = 0) or the
        prediction of step s-1, except that stream 0 is never applied here (the start frame's stream-0 noise is
        `DeviceFrames.batch(noise_std=...)`'s).  The predictions themselves stay clean, and the gradient through each
        perturbed frame is the identity, so they and the gradients equal those of the chain of one-step `rollout`
        calls on frames perturbed with `add_input_noise`.  It costs one launch and keeps one more frame per noisy step.
        noise=None, or std 0, runs exactly what runs without it.  Raises ValueError for a malformed record (see
        `check_rollout_noise`).

        teacher = TeacherForcing(frames, flags) is scheduled sampling: step s >= 1 of sample b is fed the true frame
        frames[s - 1][b] where flags[s - 1][b] is set, else the prediction of step s - 1 (with `noise`, the noise of
        stream k0 + s is added to whichever frame was chosen).  It is a choice of frame: a forced sample's input never
        depends on its prediction.  The gradient w.r.t. prediction s - 1 of a forced sample is then exactly the
        loss's own, and nothing flows into `frames` (a `frames` that requires grad is refused).  With all flags 0 the
        predictions and every gradient equal those without a teacher bit for bit.  It costs one launch and keeps one
        more frame per step s >= 1.  Raises ValueError for a malformed record (see `check_teacher_forcing`)."""
        batch = inputs.shape[0] if inputs.dim() == 4 else 1
        noise = check_rollout_noise(noise, batch, steps)
        teacher = check_teacher_forcing(teacher, batch, steps, *inputs.shape[-2:])
        self._require_cuda()
        if isinstance(steps, bool) or not isinstance(steps, int) or steps < 1:
            raise ValueError(f"steps must be a positive int; got {steps!r}")
        if inputs.dim() == 3:
            inputs, case_params = inputs.unsqueeze(0), case_params.unsqueeze(0)
            mask = mask.unsqueeze(0) if mask is not None else None
        inputs, case_params, mask4 = self._prep_inputs(inputs, case_params, mask)
        if noise is not None and noise.ids.device != self.device:
            raise ValueError(f"noise.ids is on {noise.ids.device}, the model on {self.device}")
        if teacher is not None and teacher.frames.device != self.device:
            raise ValueError(f"teacher.frames is on {teacher.frames.device}, the model on {self.device}")
        with torch.cuda.device(self.device):
            if self._needs_grad(inputs, case_params, mask4):
                return _RolloutFn.apply(self, inputs, mask4, case_params, steps, noise, teacher, *self.parameters())
            with torch.no_grad():
                return self._native_rollout_train(inputs, mask4, case_params, steps, noise, teacher)[0]

    def _rollout_device(self, inputs, case_params, mask4, steps) -> Tensor:
        b = inputs.shape[0]
        pk = self._pack()
        route = self._route(*inputs.shape[-2:])
        gh, gw = route.gh, route.gw
        ws, ws_bufs = self._workspace(b, route)
        seq = torch.empty(steps, b, self.out_chan, gh, gw, dtype=torch.float32, device=self.device)
        weights = self._coords(pk, gh, gw)[0]

        def rollout(x, mk, cp, out):
            route.call("rollout", C.byref(weights), x.data_ptr(), mk.data_ptr(), cp.data_ptr(), out.data_ptr(), steps,
                       C.byref(ws), b, self._stream())
        if not self.graph_rollout:
            rollout(inputs, mask4, case_params, seq)
            return seq
        # CUDA-graph replay: static buffers, one capture per (batch, steps[, grid])
        key = (b, steps, "grid", gh, gw) if route.grid else (b, steps, self.act_dtype)
        ent = self._graphs.get(key)
        if ent is None:
            s_in, s_cp, s_mk = inputs.clone(), case_params.clone(), mask4.clone()
            s_seq = torch.empty_like(seq)

            def run():
                rollout(s_in, s_mk, s_cp, s_seq)
            with side_stream(self.device):
                run()  # warm-up: sets kernel attributes / builds constant tables outside capture
                graph = capture_graph(run)
            ent = (graph, s_in, s_cp, s_mk, s_seq, ws_bufs, pk)  # the capture holds raw pointers into these
            while len(self._graphs) >= self.max_graphs:  # oldest capture (and its static buffers) goes first
                self._graphs.pop(next(iter(self._graphs)))
            self._graphs[key] = ent
        graph, s_in, s_cp, s_mk, s_seq = ent[:5]
        s_in.copy_(inputs)
        s_cp.copy_(case_params)
        s_mk.copy_(mask4)
        graph.replay()
        seq.copy_(s_seq)
        return seq

    def _rollout_host(self, inputs: Tensor, case_params: Tensor, mask: Tensor, steps: int) -> Tensor:
        """Host tensors in -> host tensors out; the result is a tensor the caller OWNS (fresh pinned memory from torch's
        caching host allocator, never a view of a reused buffer -- the reference returns fresh tensors too).

        Multi-step rollouts run `fno_rollout_host` (H2D, rollout, D2H on one stream).  A single step of a large batch --
        the per-step host round trip that `bench.py`'s e2e number times -- is cut into HOST_CHUNKS equal batch chunks whose
        uploads, kernels and downloads go through three streams chained by events, so the copies of one chunk overlap the
        kernels of another (the cases are independent).  Each chunk's 14 kernel launches are replayed from a CUDA graph
        (one driver call), and the loop-invariant operands -- mask and case parameters -- stay on the device between
        calls: they are uploaded again only when the caller's tensors change (pointer / version / shape)."""
        lib = _lib.load()
        b = inputs.shape[0]
        if inputs.dim() == 4 and inputs.shape[1] == self.in_chan and tuple(inputs.shape[-2:]) != (H, W):
            return self._rollout_host_grid(inputs, case_params, mask, steps)
        if tuple(inputs.shape[1:]) != (self.in_chan, H, W):
            raise ValueError(f"inputs must be (B,{self.in_chan},{H},{W})")
        mask3 = mask.reshape(b, H, W)
        inputs = inputs.contiguous().float()
        case_params = case_params.contiguous().float()
        mask3 = mask3.contiguous().float()
        pk = self._pack()
        dev = self.device
        cur = torch.cuda.current_stream(dev)
        out = torch.empty(steps, b, self.out_chan, H, W, dtype=torch.float32, pin_memory=True)
        if not (steps == 1 and b >= 128 and b % HOST_CHUNKS == 0):
            key = ("host_io", b, steps)
            ent = self._ws_cache.get(key)
            if ent is None:
                nbytes = lib.fno_rollout_host_scratch_bytes(b, self.n_case_params, steps)
                ent = dict(dev_io=torch.empty(nbytes, dtype=torch.uint8, device=dev))
                self._ws_cache[key] = ent
            ws, _ = self._workspace(b)
            _lib.check(lib.fno_rollout_host(C.byref(pk["struct"]), inputs.data_ptr(), mask3.data_ptr(),
                                            case_params.data_ptr(), out.data_ptr(), steps, C.byref(ws),
                                            ent["dev_io"].data_ptr(), b, self._act_code(), self._stream()),
                       "fno_rollout_host")
            cur.synchronize()
            return out

        cb = b // HOST_CHUNKS
        key = ("host_chunked", b, self.act_dtype, self.fused_block)
        ent = self._ws_cache.get(key)
        if ent is None or ent["pk"] is not pk:
            ent = dict(
                pk=pk,
                d_in=[torch.empty(cb, self.in_chan, H, W, dtype=torch.float32, device=dev) for _ in range(HOST_CHUNKS)],
                d_mask=torch.empty(b, 1, H, W, dtype=torch.float32, device=dev),
                d_cp=torch.empty(b, max(self.n_case_params, 1), dtype=torch.float32, device=dev),
                d_out=[torch.empty(cb, self.out_chan, H, W, dtype=torch.float32, device=dev) for _ in range(HOST_CHUNKS)],
                streams=[torch.cuda.Stream(device=dev) for _ in range(3)],
                ev_in=[torch.cuda.Event() for _ in range(HOST_CHUNKS)],
                ev_cmp=[torch.cuda.Event() for _ in range(HOST_CHUNKS)],
                graphs=None, inv_key=None,
            )
            self._ws_cache[key] = ent
        s_in, s_cmp, s_out = ent["streams"]
        for st in ent["streams"]:
            st.wait_stream(cur)  # weight packing etc. happened on the current stream
        inv_key = (mask3.data_ptr(), mask3._version, case_params.data_ptr(), case_params._version, tuple(mask3.shape))
        if ent["inv_key"] != inv_key:   # loop invariants: uploaded once, reused by every following step
            with torch.cuda.stream(s_in):
                ent["d_mask"].view(b, H, W).copy_(mask3, non_blocking=True)
                if self.n_case_params > 0:
                    ent["d_cp"][:, :self.n_case_params].copy_(case_params, non_blocking=True)
            ent["inv_key"] = inv_key
        if ent["graphs"] is None:   # one capture per chunk: fno_forward on the chunk's static buffers
            graphs = []
            s_cmp.wait_stream(s_in)
            with torch.cuda.stream(s_cmp):
                for c in range(HOST_CHUNKS):
                    lo = c * cb
                    ws, _ = self._workspace(cb, slot=1 + c)
                    cp_c = ent["d_cp"][lo:lo + cb]
                    assert cp_c.is_contiguous() or self.n_case_params == 0
                    if self.n_case_params not in (0, ent["d_cp"].shape[1]):
                        raise _lib.FnoNativeError("internal: case-parameter staging width")

                    def run(c=c, ws=ws, lo=lo):
                        _lib.check(lib.fno_forward(C.byref(pk["struct"]), ent["d_in"][c].data_ptr(),
                                                   ent["d_mask"][lo:lo + cb].data_ptr(),
                                                   ent["d_cp"][lo:lo + cb].data_ptr(), ent["d_out"][c].data_ptr(),
                                                   C.byref(ws), cb, self._act_code(),
                                                   C.c_void_p(s_cmp.cuda_stream)), "fno_forward")
                    run()   # warm-up outside capture (kernel attributes, constant tables)
                    graphs.append(capture_graph(run))
            ent["graphs"] = graphs
            s_cmp.synchronize()
        out2 = out.view(b, self.out_chan, H, W)
        # issue order = dependency order per chunk (upload, kernels, download): the first chunk's graph launch is already
        # queued when its upload lands (issuing all uploads first put ~20 us of host time on the step's critical path)
        for c in range(HOST_CHUNKS):
            with torch.cuda.stream(s_in):
                ent["d_in"][c].copy_(inputs[c * cb:(c + 1) * cb], non_blocking=True)
                ent["ev_in"][c].record(s_in)
            s_cmp.wait_event(ent["ev_in"][c])
            with torch.cuda.stream(s_cmp):
                ent["graphs"][c].replay()
                ent["ev_cmp"][c].record(s_cmp)
            s_out.wait_event(ent["ev_cmp"][c])
            with torch.cuda.stream(s_out):
                out2[c * cb:(c + 1) * cb].copy_(ent["d_out"][c], non_blocking=True)
        s_out.synchronize()
        return out

    def _rollout_host_grid(self, inputs: Tensor, case_params: Tensor, mask: Tensor, steps: int) -> Tensor:
        """Host tensors on a non-64x64 grid: upload, device rollout (graph-replayed like device tensors), and a copy into
        a fresh pinned tensor the caller owns."""
        b = inputs.shape[0]
        gh, gw = self._route(*inputs.shape[-2:])[:2]
        d_in, d_cp, mask4 = self._prep_inputs(inputs, case_params, mask.reshape(b, gh, gw))
        seq = self._rollout_device(d_in, d_cp, mask4, steps)
        out = torch.empty(steps, b, self.out_chan, gh, gw, dtype=torch.float32, pin_memory=True)
        out.copy_(seq, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return out
