"""Which native entry points each Fno2d path issues on each route: the 64x64 kernels (fno_X, in fp32 or bf16 storage),
the grid-generic kernels (fno_grid_X) on the 66x65 tube grid, and the grid-generic kernels on 64x64 frames with
`generic_grid_at_64`, with `graph_rollout` on and off.  The loaded library is swapped for a proxy that records every
call's entry-point name and its integer arguments (batch, h, w, act_dtype, steps, ...) and forwards it; the recorded
calls of the entry points that exist in both families are compared with a table written out by hand.  Two rules are
not the model's route: host-tensor `generate_many` on 64x64 frames runs the 64x64 kernels whatever generic_grid_at_64
says, and `DeviceFrames` picks its gather by the frames' shape."""
import ctypes as C

import numpy as np
import pytest
import torch

from cfdbench_b200 import _lib, synth

pytestmark = pytest.mark.gpu

B, K, P = 3, 2, 5      # batch, rollout steps, case parameters (cavity and tube)
N = 9                  # samples of the chained split: 3 cases of 4 frames; 6 two-step windows
HB, HC = 256, 128      # host-tensor single step: batch and chunk (HOST_CHUNKS = 2)
F32, BF16 = _lib.ACT_F32, _lib.ACT_BF16

# the entry points that come in both families, by their name without the fno_ / fno_grid_ prefix
ROUTED = {"forward", "forward_train", "backward", "backward_inputs", "rollout", "rollout_host", "rollout_forward_train",
          "rollout_backward", "bwd_partials_bytes", "gather_batch", "gather_window"}
ROUTES = {"f32": ("cavity", "float32", False), "bf16": ("cavity", "bfloat16", False), "grid": ("tube", "float32", False),
          "generic": ("cavity", "float32", True)}
PATHS = ["forward", "forward_backward", "rollout_backward", "generate_many_device", "generate_many_host_1",
         "generate_many_host_K", "batch", "rollout_batch", "train_auto_1", "train_auto_2"]


def _expected(route: str, graph: bool) -> dict:
    g = 2 if graph else 1   # a graph-replayed call is issued twice, as warm-up and under capture, then replayed
    if route in ("f32", "bf16"):
        a = F32 if route == "f32" else BF16
        return {
            "forward": [("fno_forward", (B, a))],
            "forward_backward": [("fno_forward_train", (B, a)), ("fno_bwd_partials_bytes", ()),
                                 ("fno_backward_inputs", (B, a))],
            "rollout_backward": [("fno_bwd_partials_bytes", ())] + [("fno_rollout_forward_train", (K, B, a))] * g
                                + [("fno_rollout_backward", (K, B, a))] * g,
            "generate_many_device": [("fno_rollout", (K, B, a))] * g,
            "generate_many_host_1": [("fno_forward", (HC, a))] * 4,
            "generate_many_host_K": [("fno_rollout_host", (K, B, a))],
            "batch": [("fno_gather_batch", (B, P, F32))],
            "rollout_batch": [("fno_gather_window", (B, P, F32, K, 1, N))],
            "train_auto_1": [("fno_bwd_partials_bytes", ())]
                            + [("fno_gather_batch", (B, P, F32)), ("fno_forward_train", (B, a)),
                               ("fno_backward_inputs", (B, a))] * 2,
            "train_auto_2": [("fno_bwd_partials_bytes", ())]
                            + [("fno_gather_window", (B, P, F32, K, 1, N)), ("fno_rollout", (1, B, a)),
                               ("fno_rollout_forward_train", (1, B, a)), ("fno_rollout_backward", (1, B, a))] * 2,
        }
    if route == "grid":
        return {
            "forward": [("fno_grid_forward", (B, 66, 65))],
            "forward_backward": [("fno_grid_forward_train", (B, 66, 65)), ("fno_grid_bwd_partials_bytes", (66, 65)),
                                 ("fno_grid_backward", (B, 66, 65))],
            "rollout_backward": [("fno_grid_bwd_partials_bytes", (66, 65))]
                                + [("fno_grid_rollout_forward_train", (K, B, 66, 65))] * g
                                + [("fno_grid_rollout_backward", (K, B, 66, 65))] * g,
            "generate_many_device": [("fno_grid_rollout", (K, B, 66, 65))] * g,
            "generate_many_host_1": [("fno_grid_rollout", (1, HB, 66, 65))] * g,
            "generate_many_host_K": [("fno_grid_rollout", (K, B, 66, 65))] * g,
            "batch": [("fno_grid_gather_batch", (B, P, F32, 66, 65))],
            "rollout_batch": [("fno_grid_gather_window", (B, P, F32, K, 1, N, 66, 65))],
            "train_auto_1": [("fno_grid_bwd_partials_bytes", (66, 65))]
                            + [("fno_grid_gather_batch", (B, P, F32, 66, 65)), ("fno_grid_forward_train", (B, 66, 65)),
                               ("fno_grid_backward", (B, 66, 65))] * 2,
            "train_auto_2": [("fno_grid_bwd_partials_bytes", (66, 65))]
                            + [("fno_grid_gather_window", (B, P, F32, K, 1, N, 66, 65)),
                               ("fno_grid_rollout", (1, B, 66, 65)), ("fno_grid_rollout_forward_train", (1, B, 66, 65)),
                               ("fno_grid_rollout_backward", (1, B, 66, 65))] * 2,
        }
    assert route == "generic"   # the grid-generic kernels on 64x64 frames, except host tensors and the gathers
    return {
        "forward": [("fno_grid_forward", (B, 64, 64))],
        "forward_backward": [("fno_grid_forward_train", (B, 64, 64)), ("fno_grid_bwd_partials_bytes", (64, 64)),
                             ("fno_grid_backward", (B, 64, 64))],
        "rollout_backward": [("fno_grid_bwd_partials_bytes", (64, 64))]
                            + [("fno_grid_rollout_forward_train", (K, B, 64, 64))] * g
                            + [("fno_grid_rollout_backward", (K, B, 64, 64))] * g,
        "generate_many_device": [("fno_grid_rollout", (K, B, 64, 64))] * g,
        "generate_many_host_1": [("fno_forward", (HC, F32))] * 4,
        "generate_many_host_K": [("fno_rollout_host", (K, B, F32))],
        "batch": [("fno_gather_batch", (B, P, F32))],
        "rollout_batch": [("fno_gather_window", (B, P, F32, K, 1, N))],
        "train_auto_1": [("fno_grid_bwd_partials_bytes", (64, 64))]
                        + [("fno_gather_batch", (B, P, F32)), ("fno_grid_forward_train", (B, 64, 64)),
                           ("fno_grid_backward", (B, 64, 64))] * 2,
        "train_auto_2": [("fno_grid_bwd_partials_bytes", (64, 64))]
                        + [("fno_gather_window", (B, P, F32, K, 1, N)), ("fno_grid_rollout", (1, B, 64, 64)),
                           ("fno_grid_rollout_forward_train", (1, B, 64, 64)),
                           ("fno_grid_rollout_backward", (1, B, 64, 64))] * 2,
    }


class _Recorder:
    """The loaded library, with every call recorded as (entry point, its int / int64 arguments) and forwarded."""

    def __init__(self, lib):
        self.real, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        ints = [i for i, t in enumerate(fn.argtypes or []) if t in (C.c_int, C.c_int64)]

        def call(*args):
            self.calls.append((name, tuple(int(args[i]) for i in ints)))
            return fn(*args)
        return call

    def routed(self) -> list:
        return [(name, args) for name, args in self.calls
                if name.removeprefix("fno_grid_").removeprefix("fno_") in ROUTED]


class _ChainSplit(torch.utils.data.Dataset):
    """3 cases of 4 chained frames (u, v, mask): inputs = frames[:-1], labels = frames[1:], time_step_size 1."""

    def __init__(self, problem):
        rng = np.random.default_rng(5)
        gh, gw = synth.grid(problem)
        masks = synth.make_mask(rng, 3, problem)[:, 0]
        ins, labs = [], []
        for c in range(3):
            fr = np.empty((4, 3, gh, gw), np.float32)
            fr[:, :2] = np.clip(rng.standard_normal((4, 2, gh, gw)), -3, 3)
            fr[:, 2] = masks[c]
            ins.append(fr[:-1])
            labs.append(fr[1:])
        self.inputs, self.labels = torch.from_numpy(np.concatenate(ins)), torch.from_numpy(np.concatenate(labs))
        self.case_ids = np.repeat(np.arange(3), 3)
        self.time_step_size = 1
        self.case_params = [{f"p{j}": float(rng.standard_normal()) for j in range(P)} for _ in range(3)]

    def __len__(self):
        return len(self.inputs)


def _model(route: str, graph: bool):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    problem, act_dtype, generic = ROUTES[route]
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=P, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act_dtype)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(3, n_params=P, spectral_gain=20.0).items()})
    m.generic_grid_at_64, m.graph_rollout = generic, graph
    return m.cuda(), problem


def _run(path: str, m, problem: str, rec: "_Recorder", tmp_path) -> None:
    from cfdbench_b200 import DeviceFrames, train_auto
    batch = {k: torch.from_numpy(v) for k, v in synth.make_batch(11, B, problem, with_label=False).items()}
    dev = {k: v.cuda() for k, v in batch.items()}
    x, cp, mk = dev["inputs"], dev["case_params"], dev["mask"]
    frames = DeviceFrames(_ChainSplit(problem), device="cuda") if path in ("batch", "rollout_batch") \
        or path.startswith("train_auto") else None
    torch.cuda.synchronize()
    rec.calls.clear()
    if path == "forward":
        with torch.no_grad():
            m(inputs=x, case_params=cp, mask=mk)
    elif path == "forward_backward":
        m(inputs=x, case_params=cp, mask=mk)["preds"].square().sum().backward()
    elif path == "rollout_backward":
        m.rollout(x, cp, mk, K).square().sum().backward()
    elif path == "generate_many_device":
        m.generate_many(x, cp, mk, K)
    elif path == "generate_many_host_1":
        big = {k: torch.from_numpy(v) for k, v in synth.make_batch(12, HB, problem, with_label=False).items()}
        m.generate_many(big["inputs"], big["case_params"], big["mask"], 1)
    elif path == "generate_many_host_K":
        m.generate_many(batch["inputs"], batch["case_params"], batch["mask"], K)
    elif path == "batch":
        frames.batch([0, 4, 8])
    elif path == "rollout_batch":
        frames.rollout_batch([0, 4, 7], K)
    else:
        k = 1 if path == "train_auto_1" else K
        train_auto(m, frames, frames, tmp_path, num_epochs=1, batch_size=B, eval_interval=2, rollout_steps=k,
                   rollout_grad_steps=1, generator=torch.Generator().manual_seed(0))
    torch.cuda.synchronize()


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "direct"])
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("path", PATHS)
def test_native_calls_per_path_and_route(path, route, graph, tmp_path, monkeypatch):
    m, problem = _model(route, graph)
    rec = _Recorder(_lib.load())
    monkeypatch.setattr(_lib, "_lib", rec)   # _lib.load() returns the proxy until the test ends
    _run(path, m, problem, rec, tmp_path)
    assert rec.routed() == _expected(route, graph)[path]
