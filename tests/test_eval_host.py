"""Argument checks of the grid-generic evaluation and input-batch entry points (`multistep_metrics`, `infer_multistep`,
`DeviceFrames`, `fno_grid_multistep_metrics`, `fno_grid_gather_batch`).  Everything here is rejected before any device
work is issued, so no GPU is needed."""
import ctypes as C

import numpy as np
import pytest
import torch

from cfdbench_b200 import _lib, data as cdata, infer_multistep
from cfdbench_b200.metrics import multistep_metrics


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


class _NoModel(torch.nn.Module):
    """Fails the test if infer_multistep gets as far as rolling out."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def generate_many(self, *a, **k):  # pragma: no cover
        raise AssertionError("argument checks must run before the rollout")


def _cases(shapes):
    return [torch.zeros(s) for s in shapes], [torch.zeros(5) for _ in shapes]


@pytest.mark.parametrize("grid", [(23, 64), (64, 23), (129, 66), (66, 129), (8, 8)])
def test_metrics_reject_grids_outside_range(grid):
    s, b = 2, 3
    with pytest.raises(ValueError, match="outside the supported range"):
        multistep_metrics(torch.zeros(s, b, 2, *grid), torch.zeros(s, b, *grid), torch.zeros(s, b, *grid))


@pytest.mark.parametrize("shapes", [
    ((2, 3, 2, 66, 65), (2, 3, 66, 64), (2, 3, 66, 65)),     # label_u grid
    ((2, 3, 2, 66, 65), (2, 3, 66, 65), (2, 3, 65, 66)),     # mask grid
    ((2, 3, 2, 66, 65), (2, 4, 66, 65), (2, 4, 66, 65)),     # batch
    ((2, 3, 2, 66, 65), (3, 3, 66, 65), (2, 3, 66, 65)),     # steps
    ((2, 3, 3, 66, 65), (2, 3, 66, 65), (2, 3, 66, 65)),     # channels
    ((3, 2, 66, 65), (3, 66, 65), (3, 66, 65)),              # no step axis
])
def test_metrics_reject_inconsistent_shapes(shapes):
    with pytest.raises(ValueError):
        multistep_metrics(*(torch.zeros(s) for s in shapes))


@pytest.mark.parametrize("grid", [(64, 64), (66, 65), (25, 127)])
def test_metrics_on_cpu_tensors_raise_native_error(grid):
    with pytest.raises(_lib.FnoNativeError):
        multistep_metrics(torch.zeros(2, 3, 2, *grid), torch.zeros(2, 3, *grid), torch.zeros(2, 3, *grid))


def test_infer_rejects_cases_on_different_grids():
    feats, cps = _cases([(20, 3, 66, 65), (20, 3, 66, 65), (20, 3, 64, 64)])
    with pytest.raises(ValueError, match="share one grid"):
        infer_multistep(_NoModel(), feats, cps, infer_steps=20)


def test_infer_rejects_short_cases():
    feats, cps = _cases([(20, 3, 66, 65), (19, 3, 66, 65)])
    with pytest.raises(ValueError, match="fewer than infer_steps"):
        infer_multistep(_NoModel(), feats, cps, infer_steps=20)
    with pytest.raises(_lib.FnoNativeError):   # 19 steps pass the checks, and then the rollout needs a CUDA model
        infer_multistep(_NoModel(), feats, cps, infer_steps=19)


@pytest.mark.parametrize("grid", [(23, 65), (66, 129)])
def test_infer_rejects_grids_outside_range(grid):
    feats, cps = _cases([(4, 3, *grid)] * 2)
    with pytest.raises(ValueError, match="outside the supported range"):
        infer_multistep(_NoModel(), feats, cps, infer_steps=4)


def test_infer_rejects_malformed_arguments():
    feats, cps = _cases([(4, 3, 66, 65)] * 2)
    with pytest.raises(ValueError):
        infer_multistep(_NoModel(), [], [], infer_steps=4)
    with pytest.raises(ValueError):
        infer_multistep(_NoModel(), feats, cps[:1], infer_steps=4)
    with pytest.raises(ValueError):
        infer_multistep(_NoModel(), feats, cps, infer_steps=0)
    with pytest.raises(ValueError):
        infer_multistep(_NoModel(), feats, cps, infer_steps=4, max_batch=0)
    with pytest.raises(ValueError, match=r"\(T, 3, H, W\)"):
        infer_multistep(_NoModel(), [torch.zeros(4, 2, 66, 65)] * 2, cps, infer_steps=4)
    with pytest.raises(ValueError, match=r"\(T, 3, H, W\)"):   # numpy arrays are accepted as features
        infer_multistep(_NoModel(), [np.zeros((4, 66, 65), np.float32)] * 2, cps, infer_steps=4)


class _Frames:
    def __init__(self, ins, labs=None):
        self.inputs, self.labels = ins, ins if labs is None else labs
        self.case_ids = np.zeros(ins.shape[0], np.int64)
        self.case_params = [dict(density=1.0, viscosity=0.1)]


@pytest.mark.parametrize("ins,labs", [
    (torch.zeros(5, 2, 66, 65), None),                  # no mask channel
    (torch.zeros(5, 3, 66), None),                      # 3-D
    (torch.zeros(5, 3, 66, 65), torch.zeros(5, 3, 65, 66)),
    (torch.zeros(5, 3, 66, 65), torch.zeros(4, 3, 66, 65)),
    (torch.zeros(5, 3, 23, 65), None),                  # grid outside 24..128
    (torch.zeros(5, 3, 66, 129), None),
])
def test_device_frames_reject_bad_frames(ins, labs):
    with pytest.raises(ValueError):
        cdata.DeviceFrames(_Frames(ins, labs), device="cuda")


def test_abi_rejects_bad_grid_and_arguments(lib):
    st = C.c_void_p(0)
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first
    assert lib.fno_grid_multistep_metrics(one, one, one, one, 2, 3, 66, 129, st) == 3
    assert b"outside the supported range" in lib.fno_last_error()
    assert lib.fno_grid_multistep_metrics(one, one, one, one, 2, 3, 23, 65, st) == 3
    assert lib.fno_grid_multistep_metrics(None, one, one, one, 2, 3, 66, 65, st) == 1
    assert b"fno_grid_multistep_metrics: bad argument" in lib.fno_last_error()
    assert lib.fno_grid_multistep_metrics(one, one, one, one, 0, 3, 66, 65, st) == 1
    assert lib.fno_grid_multistep_metrics(one, one, one, one, 2, 0, 66, 65, st) == 1
    assert lib.fno_grid_multistep_metrics(one, one, one, one, 65536, 3, 66, 65, st) == 1
    g = lambda n_idx=4, p=5, dt=_lib.ACT_F32, h=66, w=65, fin=one: lib.fno_grid_gather_batch(  # noqa: E731
        fin, one, one, one, one, n_idx, p, dt, one, one, one, one, h, w, st)
    assert g(h=130) == 3 and b"fno_grid_gather_batch" in lib.fno_last_error()
    assert g(w=20) == 3
    assert g(fin=None) == 1 and b"fno_grid_gather_batch: bad argument" in lib.fno_last_error()
    assert g(n_idx=0) == 1
    assert g(p=-1) == 1
    assert g(p=17) == 1
    assert g(dt=2) == 1
