"""Single-step evaluation on the device: `fno_eval_sums` against float64, and `evaluate_auto` -- the batched replacement
of the reference's `train_auto.evaluate` (src/train_auto.py:61-148) -- against that loop restated with the same drop-in
model and against the reference's own `evaluate`."""
import copy
import ctypes as C
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from test_data_pipeline import _collate

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.path.join(ROOT, "oracle", "_ref", "src")
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _at(n, offset):
    """A CUDA float32 tensor of n elements that starts `offset` floats into a larger, sentinel-filled buffer, with
    `offset` guard floats on either side."""
    buf = torch.full((n + 2 * offset,), SENTINEL, device="cuda")
    return buf, buf[offset:offset + n]


def _guards_intact(buf, offset):
    return bool((buf[:offset] == SENTINEL).all()) and bool((buf[buf.numel() - offset:] == SENTINEL).all())


def _holed_masks(rng, b, gh, gw):
    """(b, 1, H, W) binary masks with holes: synth's cylinder masks at 64x64, the same disc-plus-walls pattern scaled to
    any other grid."""
    if (gh, gw) == (64, 64):
        return synth.make_mask(rng, b, "cylinder")
    hh, ww = np.meshgrid(np.arange(gh), np.arange(gw), indexing="ij")
    mask = np.ones((b, 1, gh, gw), np.float32)
    for i in range(b):
        r = rng.uniform(0.06, 0.12) * min(gh, gw)
        ch, cw = rng.uniform(0.25, 0.75) * gh, rng.uniform(0.2, 0.6) * gw
        mask[i, 0][(hh - ch) ** 2 + (ww - cw) ** 2 <= r * r] = 0.0
        mask[i, 0, 0, :] = mask[i, 0, gh - 1, :] = mask[i, 0, :, 0] = 0.0
    return mask


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("grid", [(64, 64), (66, 65), (24, 24), (128, 128), (25, 27)])
@pytest.mark.parametrize("b", [1, 3, 70])
def test_eval_sums_kernel_against_float64(lib, grid, b):
    gh, gw = grid
    rng = np.random.default_rng(gh * 1000 + gw + b)
    preds = rng.standard_normal((b, 2, gh, gw)).astype(np.float32)   # used as given: the kernel must not mask it
    label = rng.standard_normal((b, 2, gh, gw)).astype(np.float32)
    inputs = rng.standard_normal((b, 2, gh, gw)).astype(np.float32)
    mask = _holed_masks(rng, b, gh, gw)
    assert 0 < mask.mean() < 1

    n = b * 2 * gh * gw
    views = [_at(n, 1)[1], _at(n, 1)[1], _at(n // 2, 3)[1], _at(n, 1)[1]]   # one float past an aligned start
    for v, a in zip(views, (preds, label, mask, inputs)):
        v.copy_(torch.from_numpy(a.reshape(-1)))
    outs = []
    for _ in range(2):
        buf, sums = _at(b * 6, 5)
        assert lib.fno_eval_sums(*(v.data_ptr() for v in views), sums.data_ptr(), b, gh, gw, _stream()) == 0, \
            lib.fno_last_error()
        torch.cuda.synchronize()
        assert _guards_intact(buf, 5)
        outs.append(sums.clone())
    assert torch.equal(outs[0], outs[1])   # a repeated launch is bit-identical

    p, lab, m, x = (a.astype(np.float64) for a in (preds, label, mask, inputs))
    lm = lab * m
    ref = np.stack([((p - lm) ** 2).sum(axis=(1, 2, 3)), np.abs(p - lm).sum(axis=(1, 2, 3)), (lm ** 2).sum(axis=(1, 2, 3)),
                    ((x[:, 0] - lab[:, 0]) ** 2).sum(axis=(1, 2)), np.abs(x[:, 0] - lab[:, 0]).sum(axis=(1, 2)),
                    (lab[:, 0] ** 2).sum(axis=(1, 2))], axis=-1)
    got = outs[0].view(b, 6).double().cpu().numpy()
    err = np.abs(got - ref) / np.abs(ref)
    print(f"eval_sums {gh}x{gw} B={b}: max rel err per sum {err.max(axis=0)}")
    assert err.max() <= 2e-5


# ------------------------------------------------------------------------------------------------ evaluate_auto
class _AutoSplit(torch.utils.data.Dataset):
    """Attributes and __getitem__ of the reference's auto datasets (`.inputs`, `.labels` (N, 3, H, W) with the mask as
    channel 2, `.case_ids`, `.case_params` dicts; src/dataset/cavity.py:283-331), filled with synth's fields and masks
    (cylinder: a hole per sample; tube: 66x65 with the wall rows and the inlet column zeroed)."""

    def __init__(self, n, problem="cavity", seed=0, n_cases=5):
        rng = np.random.default_rng(seed)
        gh, gw = synth.grid(problem)
        mask = synth.make_mask(rng, n, problem)[:, 0]
        ins = np.empty((n, 3, gh, gw), np.float32)
        labs = np.empty((n, 3, gh, gw), np.float32)
        for a in (ins, labs):
            a[:, :2] = np.clip(rng.standard_normal((n, 2, gh, gw)), -3, 3)
            a[:, 2] = mask
        self.inputs, self.labels = torch.from_numpy(ins), torch.from_numpy(labs)
        self.case_ids = np.sort(rng.integers(0, n_cases, n))
        p = synth.n_case_params(problem)
        self.case_params = [dict(rotated=c % 2, **{f"p{j}": float(rng.standard_normal()) for j in range(p)}, dx=0.1)
                            for c in range(n_cases)]

    def __len__(self):
        return len(self.inputs)

    def __getitem__(self, idx):
        return self.inputs[idx], self.labels[idx], self.case_params[self.case_ids[idx]]


def _model(problem, act_dtype="float32", seed=3, loss="nmse"):
    from cfdbench_b200 import Fno2d
    from cfdbench_b200.loss import loss_name_to_fn
    p = synth.n_case_params(problem)
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn(loss), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act_dtype)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(seed, n_params=p, spectral_gain=20.0).items()})
    return m.cuda()


def _reference_loop(model, ds, batch_size):
    """The reference's evaluate (src/train_auto.py:61-148) restated without its plots: DataLoader + collate_fn and
    .cuda(), the input loss and the forward with label, .cpu().tolist() of every score, preds.view(-1, 1, h, w).cpu()."""
    loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=False,
                                         collate_fn=lambda b: {k: v.cuda() for k, v in _collate(b).items()})
    scores = {name: [] for name in model.loss_fn.get_score_names()}
    input_scores = copy.deepcopy(scores)
    all_preds = []
    model.eval()
    with torch.inference_mode():
        for batch in loader:
            inputs, labels = batch["inputs"], batch["label"]
            input_loss = model.loss_fn(labels=labels[:, :1], preds=inputs[:, :1])
            for k in input_scores:
                input_scores[k].append(input_loss[k].cpu().tolist())
            outputs = model(**batch)
            preds = outputs["preds"].view(-1, 1, *labels.shape[2:])
            for k in scores:
                scores[k].append(outputs["loss"][k].cpu().tolist())
            all_preds.append(preds.cpu().detach())
    mean = {}
    for k in scores:
        mean[k] = np.mean(scores[k])
        mean[f"input_{k}"] = np.mean(input_scores[k])
    return dict(preds=torch.cat(all_preds, dim=0), scores=dict(mean=mean, all=scores))


def _max_rel_diff(got, ref):
    """Largest relative difference over every per-batch and mean score; the key orders must agree."""
    assert list(got["mean"]) == list(ref["mean"]) and list(got["all"]) == list(ref["all"])
    worst = 0.0
    for k in ref["all"]:
        assert len(got["all"][k]) == len(ref["all"][k])
        for g, r in zip(got["all"][k], ref["all"][k]):
            worst = max(worst, abs(g - r) / abs(r))
    for k in ref["mean"]:
        worst = max(worst, abs(got["mean"][k] - ref["mean"][k]) / abs(ref["mean"][k]))
    return worst


@pytest.mark.parametrize("problem,act_dtype", [("cavity", "float32"), ("cavity", "bfloat16"), ("cylinder", "float32"),
                                               ("tube", "float32")])
def test_evaluate_auto_matches_reference_loop(problem, act_dtype):
    from cfdbench_b200 import DeviceFrames, evaluate_auto
    n = 37   # short last batch at every batch size below
    ds = _AutoSplit(n, problem, seed=11)
    gh, gw = synth.grid(problem)
    m = _model(problem, act_dtype)
    frames = DeviceFrames(ds, device="cuda")
    for batch_size in (1, 2, 16):
        ref = _reference_loop(m, ds, batch_size)
        for data in (ds, frames):
            got = evaluate_auto(m, data, batch_size=batch_size, max_batch=16)
            assert got["preds"].device.type == "cpu" and got["preds"].dtype == torch.float32
            assert tuple(got["preds"].shape) == (2 * n, 1, gh, gw)
            assert torch.equal(got["preds"], ref["preds"])
            assert all(len(v) == -(-n // batch_size) for v in got["scores"]["all"].values())
            json.dumps(got["scores"])
            worst = _max_rel_diff(got["scores"], ref["scores"])
            print(f"{problem} {act_dtype} batch_size={batch_size}: max rel score diff {worst:.3e}")
            assert worst <= 2e-6


@pytest.mark.parametrize("problem,act_dtype", [("cavity", "bfloat16"), ("tube", "float32")])
def test_evaluate_auto_does_not_depend_on_max_batch(problem, act_dtype):
    from cfdbench_b200 import DeviceFrames, evaluate_auto
    m = _model(problem, act_dtype, seed=4)
    frames = DeviceFrames(_AutoSplit(23, problem, seed=2), device="cuda")
    outs = [evaluate_auto(m, frames, batch_size=2, max_batch=mb) for mb in (1, 7, 256)]
    for o in outs[1:]:
        assert torch.equal(o["preds"], outs[0]["preds"])
        assert o["scores"] == outs[0]["scores"]


def test_evaluate_auto_keeps_the_models_storage_mode_check():
    """A bf16-storage model runs 64x64 only: on the tube grid it raises the model's own ValueError, before any work."""
    from cfdbench_b200 import evaluate_auto
    m = _model("tube", "bfloat16")
    with pytest.raises(ValueError, match="act_dtype"):
        evaluate_auto(m, _AutoSplit(3, "tube"))


def test_evaluate_auto_state_syncs_and_memory():
    from cfdbench_b200 import DeviceFrames, evaluate_auto
    m = _model("cavity", seed=6)
    m.train()
    before = {k: v.detach().clone() for k, v in m.state_dict().items()}
    n, max_batch = 64, 16
    small = DeviceFrames(_AutoSplit(n, "cavity", seed=1), device="cuda")
    large = DeviceFrames(_AutoSplit(4 * n, "cavity", seed=1), device="cuda")
    out = evaluate_auto(m, small, batch_size=16, max_batch=max_batch)   # also warms the model's workspace and packs
    assert not m.training   # model.eval(), as the reference
    assert not out["preds"].requires_grad and out["preds"].grad_fn is None
    assert not torch.is_inference(out["preds"])   # a normal tensor, as the reference's torch.cat returns
    assert all(p.grad is None for p in m.parameters())
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k

    # one synchronisation per call
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            evaluate_auto(m, small, batch_size=16, max_batch=max_batch)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
    syncs = [str(w.message) for w in caught if "called a synchronizing CUDA operation" in str(w.message)]
    print("synchronising operations:", len(syncs), syncs[:3])
    assert len(syncs) == 1

    # device memory: one chunk at a time; the only part that grows with N is the (N, 6) float32 sums
    rises = []
    for frames in (small, large):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        evaluate_auto(m, frames, batch_size=16, max_batch=max_batch)
        torch.cuda.synchronize()
        rises.append(torch.cuda.max_memory_allocated() - base)
    print(f"peak rise during the call: N={n}: {rises[0]} B, N={4 * n}: {rises[1]} B, sums difference {24 * 3 * n} B")
    assert rises[1] - rises[0] <= 24 * 3 * n + 1024


_REF_EVALUATE = r"""
import json, sys
from pathlib import Path
import torch
sys.path.insert(0, {root!r})
sys.path.insert(0, {tests!r})
from cfdbench_b200 import runner
runner.install({src!r}, stub_missing=True)
import train_auto
from cfdbench_b200.metrics import evaluate_auto
from test_gpu_eval_auto import _AutoSplit, _model
out = {{}}
for problem in ("cavity", "tube"):
    m = _model(problem, seed=5)
    ds = _AutoSplit(9, problem, seed=3)
    for bs in (1, 4):
        ref = train_auto.evaluate(m, ds, Path({tmp!r}) / f"{{problem}}_{{bs}}", batch_size=bs)
        ours = evaluate_auto(m, ds, batch_size=bs, max_batch=4)
        out[f"{{problem}}_{{bs}}"] = dict(
            ref=dict(mean={{k: float(v) for k, v in ref["scores"]["mean"].items()}}, all=ref["scores"]["all"]),
            ours=ours["scores"], preds_equal=torch.equal(ref["preds"], ours["preds"]),
            shapes=[list(ref["preds"].shape), list(ours["preds"].shape)])
print("RESULT " + json.dumps(out))
"""


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF_SRC, "models", "fno")),
                    reason="oracle/_ref/src (installed by __graft_entry__.build()) is not present")
def test_evaluate_auto_matches_reference_evaluate(tmp_path):
    env = {**os.environ, "PYTHONDONTWRITEBYTECODE": "1"}
    code = _REF_EVALUATE.format(root=ROOT, tests=os.path.join(ROOT, "tests"), src=REF_SRC, tmp=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    out = json.loads(line[len("RESULT "):])
    assert sorted(out) == ["cavity_1", "cavity_4", "tube_1", "tube_4"]
    for key, o in out.items():
        assert o["preds_equal"], key
        assert o["shapes"][0] == o["shapes"][1]
        worst = _max_rel_diff(o["ours"], o["ref"])
        print(f"{key}: max rel diff against the reference's evaluate {worst:.3e}")
        assert worst <= 1e-5, key
