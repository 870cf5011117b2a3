"""Checkpoint selection by rollout error on the device: `fno_[grid_]window_metrics` and `evaluate_rollout_auto` bit for
bit against the eager composition a user writes (gather the start samples, `generate_many`, gather S label frames, the
multistep-metrics kernel), chunk invariance, a float64 bound on the kernel's sums, the memory of one chunk, and
`train_auto(dev_rollout_steps=S)`: training bit-identical to the run without it, the files the reference's
get_best_ckpt reads, and the chain check of the dev split."""
import copy
import json

import numpy as np
import pytest
import torch

from cfdbench_b200 import DeviceFrames, evaluate_rollout_auto, rollout_windows, synth, train_auto
from cfdbench_b200.metrics import _launch_metrics, _window_sums, rollout_scores
from oracle import error_bounds as eb
from test_gpu_eval_auto import _model

pytestmark = pytest.mark.gpu


class _Chained:
    """A split laid out as the reference's auto datasets lay it out, on any grid: per case T_c frames (u, v, mask),
    inputs = frames[:-s], labels = frames[s:], the cases one after another, a `time_step_size`.  Each case has its own
    mask with holes, and the frames' u, v are zero where the mask is."""

    def __init__(self, lengths, grid=(64, 64), s=1, seed=0, p=5):
        rng = np.random.default_rng(seed)
        gh, gw = grid
        ins, labs, ids = [], [], []
        for c, t in enumerate(lengths):
            fr = np.empty((t, 3, gh, gw), np.float32)
            fr[:, 2] = (rng.random((gh, gw)) > 0.15).astype(np.float32)
            fr[:, :2] = np.clip(rng.standard_normal((t, 2, gh, gw)), -3, 3) * fr[:1, 2:3]
            ins.append(fr[:-s])
            labs.append(fr[s:])
            ids += [c] * (t - s)
        self.inputs, self.labels = torch.from_numpy(np.concatenate(ins)), torch.from_numpy(np.concatenate(labs))
        self.case_ids = np.asarray(ids)
        self.time_step_size = s
        self.case_params = [{f"p{j}": float(rng.standard_normal()) for j in range(p)} for _ in lengths]

    def __len__(self):
        return len(self.inputs)


def _grid_model(grid, act_dtype="float32"):
    """The 64x64 problems' model (5 case parameters) on any grid: Fno2d takes the grid from its inputs."""
    return _model("cavity", act_dtype=act_dtype)


def _eager_sums(model, frames, starts, S, s):
    """The composition without the new kernel: (S, B, 3) float32 sums of the multistep-metrics kernel on the gathered
    predictions, label u planes and start masks."""
    starts = torch.as_tensor(starts, dtype=torch.int64)
    with torch.no_grad():
        b0 = frames.batch(starts)
        preds = torch.stack(model.generate_many(b0["inputs"], b0["case_params"], b0["mask"], S))
        label_u = torch.stack([frames.batch(starts + k * s)["label"][:, 0] for k in range(S)])
        mask = b0["mask"][:, 0].expand(S, -1, -1, -1).contiguous()
        sums = torch.empty(S, starts.numel(), 3, device="cuda")
        _launch_metrics(preds, label_u.contiguous(), mask, sums)
    return sums, preds


CONFIGS = [  # (grid, frame dtype, storage mode of the model)
    ((64, 64), torch.float32, "float32"),
    ((64, 64), torch.bfloat16, "float32"),
    ((64, 64), torch.float32, "bfloat16"),
    ((66, 65), torch.float32, "float32"),
    ((25, 127), torch.float32, "float32"),   # odd H*W: every other plane only 4-byte aligned
]


@pytest.mark.parametrize("grid, frame_dtype, act_dtype", CONFIGS)
@pytest.mark.parametrize("S, s", [(1, 1), (3, 2), (20, 1), (20, 2)])
def test_bit_identical_to_the_eager_composition(grid, frame_dtype, act_dtype, S, s):
    ds = _Chained((45, 9, 50), grid, s=s, seed=S * 10 + s)
    frames = DeviceFrames(ds, device="cuda", frame_dtype=frame_dtype)
    model = _grid_model(grid, act_dtype)
    windows = rollout_windows(ds.case_ids, S, s)
    assert windows.size > 0
    want, _ = _eager_sums(model, frames, windows, S, s)
    want = want.double().cpu().numpy()
    with torch.inference_mode():
        got = _window_sums(model, frames, windows, S, s, max_batch=256)
    assert got.shape == (S, windows.size, 3)
    assert np.array_equal(got, want), np.abs(got - want).max()
    res = evaluate_rollout_auto(model, frames, S)
    assert res == rollout_scores(want, grid[0] * grid[1])
    assert res["windows"] == windows.size and len(res["steps"]) == S
    assert np.isfinite(res["loss"]) and res["loss"] > 0
    # the reference dataset object gives the same result as its DeviceFrames (fp32 frames)
    if frame_dtype == torch.float32:
        assert evaluate_rollout_auto(model, ds, S) == res


def test_chunk_invariance():
    ds = _Chained((40,) * 9, (64, 64), s=1, seed=5)
    frames = DeviceFrames(ds, device="cuda")
    assert rollout_windows(ds.case_ids, 3, 1).size == 333
    model = _model("cavity")
    res = [evaluate_rollout_auto(model, frames, 3, max_batch=mb) for mb in (64, 256, 512)]
    assert res[0] == res[1] == res[2] and res[0]["windows"] == 333


@pytest.mark.parametrize("grid", [(64, 64), (66, 65)])
def test_sums_within_float64_bound(grid):
    """The kernel's sums against float64 numpy on the GPU's own predictions and frames.  Per sum the bound is the
    accumulation's kappa(H*W) on the sum of |terms| plus the rounding of d = p m - l m in float32 (at most 2^-23 (|d| +
    |l m|) per pixel, carried into d^2 by 2 |d|)."""
    S, s = 5, 1
    ds = _Chained((20, 30), grid, s=s, seed=11)
    frames = DeviceFrames(ds, device="cuda")
    model = _model("cavity")
    windows = rollout_windows(ds.case_ids, S, s)
    with torch.inference_mode():
        got = _window_sums(model, frames, windows, S, s, max_batch=256)
    _, preds = _eager_sums(model, frames, windows, S, s)
    p = preds[:, :, 0].double().cpu().numpy()                                     # (S, B, H, W)
    fin, fout = ds.inputs.double().numpy(), ds.labels.double().numpy()
    m = fin[windows, 2][None]                                                      # (1, B, H, W)
    l = np.stack([fout[windows + k * s, 0] for k in range(S)])
    pm, lm = p * m, l * m
    d = pm - lm
    ref = np.stack([(d * d).sum((2, 3)), (lm * lm).sum((2, 3)), np.abs(d).sum((2, 3))], -1)
    k = eb.kappa(grid[0] * grid[1])
    rep = 2.0 ** -23 * (np.abs(d) + np.abs(lm))
    bound = np.stack([k * (d * d).sum((2, 3)) + (2 * np.abs(d) * rep).sum((2, 3)),
                      k * (lm * lm).sum((2, 3)) + (2 * np.abs(lm) * 2.0 ** -24 * np.abs(lm)).sum((2, 3)),
                      k * np.abs(d).sum((2, 3)) + rep.sum((2, 3))], -1)
    err = np.abs(got - ref)
    assert (err <= bound).all(), (err / bound).max()
    assert (ref[..., 1] > 0).all()


def test_one_chunk_allocates_no_label_sequence():
    """Peak memory of one chunk: the (S, B, 2, H, W) predictions, the gathered batch and the sums, nothing of the size
    of an (S, B, H, W) label sequence (S B H W floats = 21 MB here)."""
    S, B = 20, 64
    ds = _Chained((B + S,) + (B + S,), (64, 64), s=1, seed=2)
    frames = DeviceFrames(ds, device="cuda")
    windows = rollout_windows(ds.case_ids, S, 1)
    assert windows.size == 2 * B
    model = _model("cavity")
    evaluate_rollout_auto(model, frames, S, max_batch=B)   # warm-up: the captured rollout and its buffers
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.inference_mode():
        _window_sums(model, frames, windows[:B], S, 1, max_batch=B)
    peak = torch.cuda.max_memory_allocated() - base
    hw = 64 * 64
    preds = S * B * 2 * hw * 4
    batch = B * (2 + 2 + 1) * hw * 4 + B * 5 * 4
    sums = S * B * 3 * 4
    label_seq = S * B * hw * 4
    margin = 1 << 20
    assert peak <= preds + batch + sums + margin, (peak, preds, batch)
    assert preds + batch + sums + margin < preds + label_seq


# ------------------------------------------------------------------------------------------------ train_auto
def _get_best_ckpt(output_dir):
    """The reference's get_best_ckpt (src/utils/common.py), restated: the ckpt-* directory with the lowest dev_loss."""
    best, best_dir = float("inf"), None
    for d in sorted(output_dir.glob("ckpt-*")):
        loss = json.load(open(d / "scores.json"))["dev_loss"]
        if loss < best:
            best, best_dir = loss, d
    return best_dir


def test_train_auto_dev_rollout_steps(tmp_path):
    tr = _Chained((14, 12, 15), (64, 64), s=1, seed=21)
    dv = _Chained((12, 10), (64, 64), s=1, seed=22)
    base = _model("cavity", seed=9)
    kw = dict(num_epochs=6, lr=2e-3, batch_size=4, eval_interval=2, log_interval=1000, rollout_steps=2)
    runs = {}
    for opt in (None, 4):
        model = copy.deepcopy(base)
        g = torch.Generator().manual_seed(123)
        out = tmp_path / f"run-{opt}"
        res = train_auto(model, tr, dv, out, generator=g, dev_rollout_steps=opt, **kw)
        runs[opt] = (model, res, out)
    (m0, r0, o0), (m1, r1, o1) = runs[None], runs[4]
    # training is bit-identical with and without the option
    assert r0["train_losses"] == r1["train_losses"]
    for (n, a), b in zip(m0.named_parameters(), m1.parameters()):
        assert torch.equal(a, b), n
    for a, b in zip(m0.parameters(), m1.parameters()):
        sa, sb = r0["optimizer"].state[a], r1["optimizer"].state[b]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"])
    ckpts = sorted(p.name for p in o0.glob("ckpt-*"))
    assert ckpts == sorted(p.name for p in o1.glob("ckpt-*")) == ["ckpt-1", "ckpt-3", "ckpt-5"]
    losses = {}
    for c in ckpts:
        assert (o0 / c / "dev_scores.json").read_bytes() == (o1 / c / "dev_scores.json").read_bytes()
        assert not (o0 / c / "dev_rollout_scores.json").exists()
        s0, s1 = json.load(open(o0 / c / "scores.json")), json.load(open(o1 / c / "scores.json"))
        assert list(s0) == ["ep", "train_loss", "dev_loss", "time"]
        assert list(s1) == ["ep", "train_loss", "dev_loss", "dev_loss_single_step", "time"]
        assert s1["dev_loss_single_step"] == s0["dev_loss"] and s1["train_loss"] == s0["train_loss"]
        # dev_loss is the rollout loss of that checkpoint, reloaded into a fresh model
        fresh = _model("cavity", seed=1)
        fresh.load_state_dict(torch.load(o1 / c / "model.pt", map_location="cpu"))
        again = evaluate_rollout_auto(fresh, dv, 4)
        assert s1["dev_loss"] == again["loss"]
        assert json.load(open(o1 / c / "dev_rollout_scores.json")) == again
        losses[c] = again["loss"]
    assert _get_best_ckpt(o1).name == min(losses, key=losses.get)


def test_train_auto_refuses_a_dev_split_that_does_not_chain(tmp_path):
    tr = _Chained((10, 10), (64, 64), s=1, seed=31)
    dv = _Chained((9, 8), (64, 64), s=1, seed=32)
    perm = np.arange(len(dv))
    perm[[3, 4]] = perm[[4, 3]]
    dv.inputs = dv.inputs[perm]   # sample 3's input is no longer sample 2's label
    model = _model("cavity")
    before = [p.detach().clone() for p in model.parameters()]
    with pytest.raises(ValueError, match=r"dev_data does not chain .* sample 3's input frame is not sample 2's label"):
        train_auto(model, tr, dv, tmp_path / "out", num_epochs=2, batch_size=4, dev_rollout_steps=3)
    assert all(torch.equal(a, b) for a, b in zip(before, model.parameters()))   # no training step ran
    assert not list((tmp_path / "out").glob("ckpt-*"))
    with pytest.raises(ValueError, match=r"the split does not chain .* sample 3's input frame is not sample 2's label"):
        evaluate_rollout_auto(model, dv, 3)
    # single-step evaluation, and no rollout selection, do not need the chain
    train_auto(model, tr, dv, tmp_path / "out2", num_epochs=1, batch_size=4, eval_interval=1)
