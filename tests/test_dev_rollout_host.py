"""Checkpoint selection by rollout error (`evaluate_rollout_auto`, `train_auto(dev_rollout_steps=S)`) without a GPU: the
argument refusals, which all come before any device work, the dev windows on ragged case layouts, the host reduction
against a float64 restatement, and the declarations and argument checks of `fno_[grid_]window_metrics`."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cfdbench_b200
from cfdbench_b200 import _lib, evaluate_rollout_auto, rollout_windows, train_auto
from cfdbench_b200.metrics import rollout_scores
from test_train_auto_host import _cpu_model, _Split
from test_train_rollout_host import _TimedSplit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("fno_window_metrics", "fno_grid_window_metrics")


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


# ------------------------------------------------------------------------------------------------ C ABI
def test_new_entry_points_are_declared_and_exported(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(rf"\bint\s+{name}\s*\(", hdr), name
        assert hasattr(C.CDLL(_lib.LIB_PATH), name)
        assert name in _lib.SIGNATURES
    assert "evaluate_rollout_auto" in cfdbench_b200.__all__


def test_window_metrics_reject_bad_arguments(lib):
    st = C.c_void_p(0)
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first

    def call(grid=None, preds=one, fin=one, fout=one, starts=one, steps=3, batch=4, s=1, n=10, dtype=0, sums=one):
        args = (preds, fin, fout, starts, steps, batch, s, n, dtype, sums)
        if grid is None:
            return lib.fno_window_metrics(*args, st), b"fno_window_metrics"
        return lib.fno_grid_window_metrics(*args, *grid, st), b"fno_grid_window_metrics"
    for grid in (None, (66, 65), (25, 127)):
        for kw in (dict(preds=None), dict(fin=None), dict(fout=None), dict(starts=None), dict(sums=None), dict(steps=0),
                   dict(steps=65536), dict(batch=0), dict(batch=-1), dict(s=0), dict(n=0), dict(dtype=2), dict(dtype=-1)):
            status, name = call(grid, **kw)
            assert status == 1, (grid, kw)
            assert name + b": bad argument" in lib.fno_last_error()
    # the 64x64 kernel's vector loads: 16-byte predictions, 16-byte fp32 / 8-byte bf16 frames
    for kw in (dict(preds=C.c_void_p(24)), dict(fin=C.c_void_p(24)), dict(fout=C.c_void_p(20), dtype=1)):
        assert call(**kw)[0] == 1, kw
        assert b"aligned" in lib.fno_last_error()
    # an out-of-range grid is refused with status 3 before the other checks
    for grid in ((66, 129), (23, 65), (0, 0)):
        assert call(grid)[0] == 3, grid
        assert call(grid, preds=None)[0] == 3, grid


# ------------------------------------------------------------------------------------------------ argument refusals
def test_evaluate_rollout_auto_rejects_bad_arguments():
    m = _cpu_model()
    dv = _TimedSplit(12)
    for k in (0, -1, 2.0, True, "2", None):
        with pytest.raises(ValueError, match="steps must be a positive int"):
            evaluate_rollout_auto(m, dv, k)
    for s in (0, -2, 1.5, True):
        with pytest.raises(ValueError, match="time_step_size must be a positive int"):
            evaluate_rollout_auto(m, dv, 2, time_step_size=s)
    for mb in (0, -1, 1.0, False):
        with pytest.raises(ValueError, match="max_batch must be a positive int"):
            evaluate_rollout_auto(m, dv, 2, max_batch=mb)
    with pytest.raises(TypeError, match="Fno2d"):
        import torch
        evaluate_rollout_auto(torch.nn.Linear(2, 2), dv, 2)
    with pytest.raises(ValueError, match="needs a time_step_size"):
        evaluate_rollout_auto(m, _Split(12), 2)                  # the dataset has no time_step_size
    with pytest.raises(ValueError, match="time_step_size must be a positive int"):
        evaluate_rollout_auto(m, _TimedSplit(12, s=0), 2)        # nor a usable one
    with pytest.raises(ValueError, match="no 7-step window"):
        evaluate_rollout_auto(m, dv, 7)                          # cases of 6 samples
    with pytest.raises(ValueError, match="no 3-step window with time_step_size=3"):
        evaluate_rollout_auto(m, dv, 3, time_step_size=3)
    with pytest.raises(ValueError, match="empty"):
        evaluate_rollout_auto(m, _TimedSplit(0, n_cases=1), 1)
    with pytest.raises(ValueError, match="case parameters per sample"):
        evaluate_rollout_auto(m, _Split(4, p=3), 1, time_step_size=1)
    with pytest.raises(ValueError, match="supports"):
        evaluate_rollout_auto(m, _Split(4, 20, 64), 1, time_step_size=1)
    with pytest.raises(ValueError, match="act_dtype"):
        evaluate_rollout_auto(_cpu_model(act_dtype="bfloat16"), _Split(4, 66, 65), 1, time_step_size=1)
    # a valid set-up gets as far as the CPU model's refusal, before any device work
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        evaluate_rollout_auto(m, dv, 6)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        evaluate_rollout_auto(m, _Split(12), 1, time_step_size=1)


def test_train_auto_rejects_bad_dev_rollout_steps(tmp_path):
    out = tmp_path / "out"
    tr, dv = _Split(4), _TimedSplit(12)
    m = _cpu_model()
    for k in (0, -1, 2.0, True, False, "2"):
        with pytest.raises(ValueError, match="dev_rollout_steps must be a positive int"):
            train_auto(m, tr, dv, out, dev_rollout_steps=k)
    with pytest.raises(ValueError, match="dev_rollout_steps=2 needs a time_step_size: dev_data has none"):
        train_auto(m, tr, _Split(12), out, dev_rollout_steps=2)
    with pytest.raises(ValueError, match="time_step_size must be a positive int"):
        train_auto(m, tr, _TimedSplit(12, s=0), out, dev_rollout_steps=2)
    with pytest.raises(ValueError, match="dev_data has no 7-step window"):
        train_auto(m, tr, dv, out, dev_rollout_steps=7)
    with pytest.raises(ValueError, match="dev_data has no 3-step window with time_step_size=3"):
        train_auto(m, tr, dv, out, dev_rollout_steps=3, time_step_size=3)
    # valid set-ups get as far as the CPU model's refusal; the time_step_size argument overrides the split's
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, dv, out, dev_rollout_steps=6)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, _Split(12), out, dev_rollout_steps=2, time_step_size=1)
    assert not out.exists()   # rejected before anything was written


# ------------------------------------------------------------------------------------------------ windows
@pytest.mark.parametrize("lengths", [(1, 7, 2, 9, 3), (5,), (2, 2, 2), (11, 1, 1, 6)])
@pytest.mark.parametrize("steps, s", [(1, 1), (3, 1), (3, 2), (4, 3)])
def test_dev_windows_on_ragged_cases(lengths, steps, s):
    """Every start whose S-step window stays inside its case, in ascending order, and nothing else."""
    ids = np.repeat(np.arange(len(lengths)), lengths)
    want = [j for j in range(ids.size)
            if j + (steps - 1) * s < ids.size and all(ids[j + k * s] == ids[j] for k in range(steps))]
    got = rollout_windows(ids, steps, s)
    assert got.dtype == np.int64 and got.tolist() == want


# ------------------------------------------------------------------------------------------------ host reduction
def _restated(sums, hw):
    """rollout_scores restated with Python floats: per window mse = e/hw, nmse = mse / (l/hw), mae = a/hw (inf / nan
    where l = 0), each step the mean over the windows added in window order, loss the mean of the steps' nmse."""
    S, n, _ = sums.shape

    def div(a, b):
        if b == 0.0:
            return float("nan") if a == 0.0 else float("inf") * np.sign(a)
        return a / b
    steps = []
    for k in range(S):
        tot = dict(mse=0.0, nmse=0.0, mae=0.0)
        for i in range(n):
            e, l, a = (float(v) for v in sums[k, i])
            mse = e / hw
            tot["mse"] += mse
            tot["nmse"] += div(mse, l / hw)
            tot["mae"] += a / hw
        steps.append({key: v / n for key, v in tot.items()})
    loss = 0.0
    for st in steps:
        loss += st["nmse"]
    return dict(steps=steps, loss=loss / S, windows=n)


def _same(a, b):
    return a == b or (np.isnan(a) and np.isnan(b))


@pytest.mark.parametrize("S, n, hw", [(1, 1, 4096), (3, 7, 4096), (20, 333, 66 * 65), (2, 5, 25 * 127)])
def test_rollout_scores_match_float64_restatement(S, n, hw):
    rng = np.random.default_rng(S * 1000 + n)
    sums = np.abs(rng.standard_normal((S, n, 3))).astype(np.float32).astype(np.float64) * hw
    got, want = rollout_scores(sums, hw), _restated(sums, hw)
    assert got["windows"] == want["windows"] == n
    assert len(got["steps"]) == S
    for g, w in zip(got["steps"], want["steps"]):
        assert set(g) == {"mse", "nmse", "mae"}
        for k in g:
            assert isinstance(g[k], float) and g[k] == w[k], (k, g[k], w[k])
    assert isinstance(got["loss"], float) and got["loss"] == want["loss"]


def test_rollout_scores_of_an_all_zero_label_plane():
    """A window whose masked label plane is all zero divides by zero as the reference's get_metrics does: nmse is inf
    with an error, nan without one, and the step means and the loss carry it."""
    hw = 4096
    sums = np.array([[[2.0, 1.0, 3.0], [5.0, 0.0, 1.0]],     # step 0: window 1 has l = 0, e > 0 -> inf
                     [[2.0, 4.0, 3.0], [0.0, 0.0, 0.0]]])    # step 1: window 1 has l = 0, e = 0 -> nan
    got, want = rollout_scores(sums, hw), _restated(sums, hw)
    assert np.isinf(got["steps"][0]["nmse"]) and np.isnan(got["steps"][1]["nmse"]) and np.isnan(got["loss"])
    for g, w in zip(got["steps"], want["steps"]):
        for k in g:
            assert _same(g[k], w[k]), (k, g[k], w[k])
    assert got["steps"][0]["mse"] == (2.0 / hw + 5.0 / hw) / 2 and got["steps"][1]["mae"] == (3.0 / hw + 0.0) / 2
    only_inf = rollout_scores(sums[:1], hw)
    assert np.isinf(only_inf["loss"])
