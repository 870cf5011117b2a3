"""`evaluate_auto` (the batched replacement of the reference's `train_auto.evaluate`, src/train_auto.py:61-148) without a
GPU: the `fno_eval_sums` entry point's argument checks, the host reduction of per-sample sums to the reference's
per-batch scores, and the argument checks of `evaluate_auto`, all of which run before any device work."""
import ctypes as C
import json
import math
import os
import re

import numpy as np
import pytest
import torch

import cfdbench_b200
from cfdbench_b200 import _lib, evaluate_auto
from cfdbench_b200.loss import MseLoss
from cfdbench_b200.metrics import eval_scores

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


# ------------------------------------------------------------------------------------------------ C ABI
def test_eval_sums_is_declared_and_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read()
    assert re.search(r"\bint\s+fno_eval_sums\s*\(", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    assert hasattr(C.CDLL(_lib.LIB_PATH), "fno_eval_sums")
    assert "fno_eval_sums" in _lib.SIGNATURES
    assert lib.fno_version() == 4
    assert "evaluate_auto" in cfdbench_b200.__all__


def test_eval_sums_rejects_bad_grid_and_arguments(lib):
    st = C.c_void_p(0)
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first
    e = lambda b=3, h=66, w=65, p=one, s=one: lib.fno_eval_sums(p, one, one, one, s, b, h, w, st)  # noqa: E731
    for h, w in ((23, 65), (66, 129), (129, 64), (64, 20)):
        assert e(h=h, w=w) == 3
        assert b"fno_eval_sums" in lib.fno_last_error() and b"outside the supported range" in lib.fno_last_error()
    assert e(p=None) == 1
    assert b"fno_eval_sums: bad argument" in lib.fno_last_error()
    assert e(s=None) == 1
    assert e(b=0) == 1
    assert e(b=-2) == 1
    assert lib.fno_eval_sums(one, None, one, one, one, 3, 64, 64, st) == 1
    assert lib.fno_eval_sums(one, one, None, one, one, 3, 64, 64, st) == 1
    assert lib.fno_eval_sums(one, one, one, None, one, 3, 64, 64, st) == 1
    assert e(b=0, h=200) == 3   # the grid is checked first, as on the other grid entry points


# ------------------------------------------------------------------------------------------------ host reduction
def _evaluate_restated(sums, hw, batch_size, names):
    """float64 restatement of evaluate's arithmetic (reference src/train_auto.py:75-147): per batch, the model's
    MseLoss on (preds, label * mask) over n * 2 * hw values and the input loss on channel 0 over n * hw values; `all`
    holds the per-batch prediction scores, `mean` np.mean over batches of both."""
    def loss(e2, e1, l2, count):
        mse = e2 / count
        out = dict(mse=mse, rmse=math.sqrt(mse), mae=e1 / count)
        out["nmse"] = mse / (l2 / count)
        return out

    scores = {k: [] for k in names}
    input_scores = {k: [] for k in names}
    for lo in range(0, len(sums), batch_size):
        rows = [list(map(float, r)) for r in sums[lo:lo + batch_size]]
        n = len(rows)
        t = [math.fsum(r[k] for r in rows) for k in range(6)]
        pred, inp = loss(t[0], t[1], t[2], n * 2 * hw), loss(t[3], t[4], t[5], n * hw)
        for k in names:
            scores[k].append(pred[k])
            input_scores[k].append(inp[k])
    mean = {}
    for k in names:
        mean[k] = np.mean(scores[k])
        mean[f"input_{k}"] = np.mean(input_scores[k])
    return dict(mean=mean, all=scores)


@pytest.mark.parametrize("batch_size", [1, 2, 16])
@pytest.mark.parametrize("names", [["mse", "rmse", "mae", "nmse"], ["mse", "rmse", "mae"]])
@pytest.mark.parametrize("n,hw", [(37, 64 * 64), (41, 66 * 65), (5, 25 * 27)])
def test_scores_match_restated_evaluate(batch_size, names, n, hw):
    rng = np.random.default_rng(n * batch_size + len(names))
    sums = rng.random((n, 6)).astype(np.float32) * np.float32(hw)
    got = eval_scores(sums, hw, batch_size, names)
    ref = _evaluate_restated(sums, hw, batch_size, names)
    assert list(got) == ["mean", "all"]
    assert list(got["all"]) == names
    assert list(got["mean"]) == [x for k in names for x in (k, f"input_{k}")]
    n_batches = -(-n // batch_size)
    for k in names:
        assert len(got["all"][k]) == n_batches
        assert all(type(v) is float for v in got["all"][k])
        np.testing.assert_allclose(got["all"][k], ref["all"][k], rtol=1e-13, atol=0)
    for k, v in got["mean"].items():
        assert type(v) is float
        assert v == pytest.approx(float(ref["mean"][k]), rel=1e-13, abs=0)
    json.loads(json.dumps(got))   # dump_json takes it as is


def test_scores_short_last_batch_is_its_own_batch():
    """N = 5, batch_size = 2: batches {0,1}, {2,3}, {4}; no drop_last, and the short batch is not weighted by its size
    in the mean (np.mean over batches)."""
    hw = 64 * 64
    sums = np.zeros((5, 6), np.float32)
    sums[:, 0] = [1, 3, 5, 7, 100]
    sums[:, 2] = 4 * hw   # mean of the squared masked labels: 2
    sums[:, 3:] = 1
    got = eval_scores(sums, hw, 2, ["mse", "nmse"])
    assert got["all"]["mse"] == [4 / (4 * hw), 12 / (4 * hw), 100 / (2 * hw)]
    assert got["mean"]["mse"] == pytest.approx((4 / 4 + 12 / 4 + 100 / 2) / 3 / hw, rel=1e-15)
    assert got["all"]["nmse"] == pytest.approx([x / 2 for x in got["all"]["mse"]], rel=1e-15)


def test_scores_zero_labels_give_the_reference_inf_and_nan():
    hw = 66 * 65
    sums = np.ones((4, 6), np.float32)
    sums[0:2, 2] = 0     # batch 0: masked labels all zero, nonzero error -> nmse = inf
    sums[2:4, [0, 2]] = 0  # batch 1: zero error over zero labels -> nmse = 0 / 0 = nan
    sums[:, 5] = 0       # input labels all zero: input_nmse = inf
    with np.errstate(all="raise"):   # no floating-point warning escapes
        got = eval_scores(sums, hw, 2, ["mse", "rmse", "mae", "nmse"])
    assert got["all"]["nmse"][0] == math.inf and math.isnan(got["all"]["nmse"][1])
    assert math.isnan(got["mean"]["nmse"]) and got["mean"]["input_nmse"] == math.inf
    assert got["all"]["mse"][1] == 0.0 and got["all"]["mae"][1] == 2 / (2 * 2 * hw)


# ------------------------------------------------------------------------------------------------ evaluate_auto checks
class _NoModel(torch.nn.Module):
    """A CPU model that fails the test if evaluate_auto gets as far as running it."""

    def __init__(self, normalize=True):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.loss_fn = MseLoss(normalize=normalize)

    def forward(self, *a, **k):  # pragma: no cover
        raise AssertionError("argument checks must run before the forward")


class _Split:
    """The attributes evaluate_auto reads from the reference's auto datasets."""

    def __init__(self, ins, labs=None, case_ids=None):
        self.inputs, self.labels = ins, ins.clone() if labs is None else labs
        self.case_ids = np.zeros(ins.shape[0], np.int64) if case_ids is None else case_ids
        self.case_params = [dict(density=1.0, viscosity=0.1)]


def test_evaluate_rejects_bad_batch_sizes():
    ds = _Split(torch.zeros(5, 3, 64, 64))
    for bs, mb in ((0, 256), (-1, 256), (2, 0), (2, -3)):
        with pytest.raises(ValueError, match="positive"):
            evaluate_auto(_NoModel(), ds, batch_size=bs, max_batch=mb)


def test_evaluate_rejects_unknown_score_names():
    class _Loss(MseLoss):
        def get_score_names(self):
            return ["mse", "mre"]

    m = _NoModel()
    m.loss_fn = _Loss(normalize=False)
    with pytest.raises(ValueError, match="mre"):
        evaluate_auto(m, _Split(torch.zeros(5, 3, 64, 64)))


@pytest.mark.parametrize("ins,labs", [
    (torch.zeros(5, 2, 66, 65), None),                       # no mask channel
    (torch.zeros(5, 3, 66), None),                           # 3-D
    (torch.zeros(5, 3, 66, 65), torch.zeros(5, 3, 65, 66)),  # label grid
    (torch.zeros(5, 3, 66, 65), torch.zeros(4, 3, 66, 65)),  # label count
    (torch.zeros(5, 3, 23, 65), None),                       # grid outside 24..128
    (torch.zeros(5, 3, 66, 129), None),
])
def test_evaluate_rejects_malformed_frames(ins, labs):
    with pytest.raises(ValueError):
        evaluate_auto(_NoModel(), _Split(ins, labs))


def test_evaluate_rejects_other_malformed_data():
    with pytest.raises(ValueError):
        evaluate_auto(_NoModel(), object())
    with pytest.raises(ValueError):
        evaluate_auto(_NoModel(), _Split(torch.zeros(5, 3, 64, 64), case_ids=np.zeros(4, np.int64)))
    with pytest.raises(ValueError, match="empty"):
        evaluate_auto(_NoModel(), _Split(torch.zeros(0, 3, 64, 64)))


@pytest.mark.parametrize("grid", [(64, 64), (66, 65), (25, 27)])
@pytest.mark.parametrize("normalize", [True, False])
def test_evaluate_on_cpu_model_raises_native_error(grid, normalize):
    with pytest.raises(_lib.FnoNativeError, match="CUDA"):
        evaluate_auto(_NoModel(normalize), _Split(torch.zeros(3, 3, *grid)), batch_size=2, max_batch=2)
