"""Gradient-norm clipping and the EMA of the weights (`FusedAdam(max_grad_norm=..., ema_decay=...)`,
`train_auto(max_grad_norm=..., ema_decay=...)`) without a GPU: argument validation, the EMA decay table against a float64
restatement of diffusers' `EMAModel.get_decay`, the new entry points' declarations and argument checks, and a state_dict
with "ema" loading into torch.optim.Adam."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from cfdbench_b200 import FusedAdam, _lib, train_auto
from test_train_auto_host import _cpu_model, _Split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("fno_grad_norm", "fno_adam_step_ex", "fno_adam_step_dev_ex", "fno_ema_decays")


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


# ------------------------------------------------------------------------------------------------ argument validation
BAD_NORMS = (0, 0.0, -1.0, float("nan"), float("inf"), -float("inf"), True, "1.0", 1 + 0j, [1.0])
BAD_DECAYS = (1.0, 1, -1e-9, 1.5, float("nan"), float("inf"), False, "0.9", 0.5j, [0.9])


def test_fused_adam_rejects_bad_stabiliser_arguments():
    p = [torch.nn.Parameter(torch.zeros(3))]
    for v in BAD_NORMS:
        with pytest.raises(ValueError, match="max_grad_norm"):
            FusedAdam(p, max_grad_norm=v)
    for v in BAD_DECAYS:
        with pytest.raises(ValueError, match="ema_decay"):
            FusedAdam(p, ema_decay=v)
    for v in (1e-12, 1, 5.0, np.float32(2.5), np.float64(1e6)):
        assert FusedAdam(p, max_grad_norm=v).max_grad_norm == float(v)
    for v in (0, 0.0, 0.9999, np.float64(0.5)):
        assert FusedAdam(p, ema_decay=v).ema_decay == float(v)
    opt = FusedAdam(p)
    assert opt.max_grad_norm is None and opt.ema_decay is None and opt.last_grad_norm is None


def test_train_auto_rejects_bad_stabiliser_arguments(tmp_path):
    out = tmp_path / "out"
    m, tr, dv = _cpu_model(), _Split(4), _Split(3)
    for v in BAD_NORMS:
        with pytest.raises(ValueError, match="max_grad_norm"):
            train_auto(m, tr, dv, out, max_grad_norm=v)
    for v in BAD_DECAYS:
        with pytest.raises(ValueError, match="ema_decay"):
            train_auto(m, tr, dv, out, ema_decay=v)
    # valid values get as far as the CPU-model refusal, the last check before device work
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, dv, out, max_grad_norm=1.0, ema_decay=0.999)
    assert not out.exists()


# ------------------------------------------------------------------------------------------------ the EMA decay table
def _get_decay(optimization_step, decay, min_decay=0.0, update_after_step=0, use_ema_warmup=True, inv_gamma=1.0,
               power=3 / 4):
    """diffusers' EMAModel.get_decay (training_utils.py), in float64, with train_diffusers.py's configuration."""
    step = max(0, optimization_step - update_after_step - 1)
    if step <= 0:
        return 0.0
    if use_ema_warmup:
        cur = 1 - (1 + step / inv_gamma) ** -power
    else:
        cur = (1 + step) / (10 + step)
    cur = min(cur, decay)
    return max(cur, min_decay)


@pytest.mark.parametrize("decay", [0.9999, 0.999, 0.9, 0.5, 0.0])
def test_ema_decays_match_diffusers_get_decay(lib, decay):
    """EMAModel.step increments optimization_step and then calls get_decay, so Adam's step t uses get_decay(t)."""
    n = 20_000
    out = np.empty(n, np.float32)
    assert lib.fno_ema_decays(decay, 1, n, out.ctypes.data) == 0
    ref = np.asarray([_get_decay(t, decay) for t in range(1, n + 1)])
    assert out[0] == 0.0   # the EMA equals the weights after the first step
    assert np.array_equal(out, ref.astype(np.float32))   # the float32 rounding of the float64 value
    assert np.all(out <= np.float32(decay)) and np.all(np.diff(out) >= 0)
    if decay > 0.5:   # the warmup has reached the cap well inside the table
        t_cap = math.ceil((1 - decay) ** (-4 / 3))
        if t_cap < n:
            assert out[-1] == np.float32(decay)
    tail = np.empty(100, np.float32)
    assert lib.fno_ema_decays(decay, 5001, 100, tail.ctypes.data) == 0
    assert np.array_equal(tail, out[5000:5100])


# ------------------------------------------------------------------------------------------------ C ABI
def test_new_entry_points_are_declared_and_exported(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read(), flags=re.S)
    for name in NEW + ("fno_grad_norm_scratch_bytes",):
        assert re.search(rf"\b(int|size_t)\s+{name}\s*\(", hdr), name
        assert hasattr(C.CDLL(_lib.LIB_PATH), name)
        assert name in _lib.SIGNATURES
    assert re.search(rf"#define FNO_GRAD_NORM_MAX_TABLES {_lib.GRAD_NORM_MAX_TABLES}\b", hdr)
    assert lib.fno_grad_norm_scratch_bytes() >= 8 * 2


def test_new_entry_points_reject_bad_arguments(lib):
    st = C.c_void_p(0)
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first
    t = _lib.FnoAdamTensors()
    t.count = 1
    t.param[0] = t.grad[0] = t.exp_avg[0] = t.exp_avg_sq[0] = 16
    t.n[0] = 8
    bad_tabs = []
    for field, v in (("n", 0), ("count", _lib.ADAM_MAX_TENSORS + 1), ("count", -1), ("grad", None), ("param", None)):
        b = _lib.FnoAdamTensors.from_buffer_copy(t)
        if field == "count":
            b.count = v
        else:
            getattr(b, field)[0] = v
        bad_tabs.append(b)

    def norm(tabs=(t,), n=None, max_norm=1.0, out=one, scratch=one, log=None, n_log=0, cur=None):
        arr = (_lib.FnoAdamTensors * max(len(tabs), 1))(*tabs)
        return lib.fno_grad_norm(arr if tabs else None, len(tabs) if n is None else n, max_norm, out, scratch, log, n_log,
                                 cur, st)
    for kw in (dict(tabs=()), dict(n=0), dict(n=_lib.GRAD_NORM_MAX_TABLES + 1), dict(max_norm=0.0),
               dict(max_norm=-1.0), dict(max_norm=float("nan")), dict(max_norm=float("inf")), dict(out=None),
               dict(scratch=None), dict(scratch=C.c_void_p(20)), dict(log=one, n_log=4), dict(log=one, cur=one),
               *[dict(tabs=(t, b)) for b in bad_tabs[:4]]):   # of a table it reads only count, grad and n
        assert norm(**kw) == 1, kw
        assert b"fno_grad_norm" in lib.fno_last_error()

    ema = (C.c_void_p * 1)(16)
    no_ema = (C.c_void_p * 1)(None)

    def ex(tab=t, step=1, clip=None, ema_p=ema, decay=0.99):
        return lib.fno_adam_step_ex(C.byref(tab) if tab is not None else None, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, clip,
                                    ema_p, decay, st)
    for kw in (dict(tab=None), dict(step=0), dict(decay=1.0), dict(decay=-0.1), dict(decay=float("nan")),
               dict(ema_p=no_ema), *[dict(tab=b) for b in bad_tabs]):
        assert ex(**kw) == 1, kw
        assert b"fno_adam_step_ex" in lib.fno_last_error()

    def dev_ex(tab=t, coef=one, n=4, cur=one, ema_p=ema, tab_d=one):
        return lib.fno_adam_step_dev_ex(C.byref(tab) if tab is not None else None, coef, n, cur, 0.9, 0.999, 1e-8, 0.0,
                                        one, ema_p, tab_d, st)
    for kw in (dict(tab=None), dict(coef=None), dict(cur=None), dict(n=0), dict(coef=C.c_void_p(20)), dict(tab_d=None),
               dict(ema_p=no_ema), *[dict(tab=b) for b in bad_tabs]):
        assert dev_ex(**kw) == 1, kw
        assert b"fno_adam_step_dev_ex" in lib.fno_last_error()

    out = (C.c_float * 4)()
    for args in ((0.9, 0, 4, out), (0.9, 1, 0, out), (0.9, 1, 4, None), (1.0, 1, 4, out), (-0.5, 1, 4, out),
                 (float("nan"), 1, 4, out)):
        assert lib.fno_ema_decays(*args) == 1, args
        assert b"fno_ema_decays" in lib.fno_last_error()


# ------------------------------------------------------------------------------------------------ state_dict
def test_state_dict_with_ema_loads_into_torch_adam():
    m = _cpu_model()
    opt = FusedAdam(m.parameters(), lr=1e-3, max_grad_norm=1.0, ema_decay=0.999)
    for p in m.parameters():
        st = opt.init_state(p)
        assert torch.equal(st["ema"], p) and st["ema"].data_ptr() != p.data_ptr() and st["ema"].dtype == p.dtype
        st["step"] += 3
        st["ema"].add_(1)
    sd = opt.state_dict()
    assert all("ema" in s for s in sd["state"].values())
    adam = torch.optim.Adam(m.parameters(), lr=1e-3)
    adam.load_state_dict(sd)
    for p in m.parameters():
        assert float(adam.state[p]["step"]) == 3
        assert torch.equal(adam.state[p]["exp_avg"], opt.state[p]["exp_avg"])
    # and back: a FusedAdam loads its own state_dict, EMA included
    again = FusedAdam(m.parameters(), lr=1e-3, ema_decay=0.999)
    again.load_state_dict(sd)
    for p in m.parameters():
        assert torch.equal(again.state[p]["ema"], opt.state[p]["ema"])
    # without ema_decay the state has no "ema" (the default state is torch.optim.Adam's)
    plain = FusedAdam(m.parameters())
    assert set(plain.init_state(next(m.parameters()))) == {"step", "exp_avg", "exp_avg_sq"}


def test_copy_ema_to():
    m, dst = _cpu_model(), _cpu_model()
    frozen = "fc2.bias"
    dict(m.named_parameters())[frozen].requires_grad_(False)
    opt = FusedAdam([p for p in m.parameters() if p.requires_grad], ema_decay=0.9)
    with pytest.raises(ValueError, match="do not match"):
        opt.copy_ema_to(dst)   # the optimizer holds one parameter fewer
    opt = FusedAdam(m.parameters(), ema_decay=0.9)
    for name, p in m.named_parameters():
        if p.requires_grad:
            opt.init_state(p)["ema"].fill_(3.0)
    opt.copy_ema_to(dst)
    for (name, a), b in zip(m.named_parameters(), dst.parameters()):
        assert torch.equal(b, a if name == frozen else torch.full_like(a, 3.0)), name
    with pytest.raises(ValueError, match="ema_decay"):
        FusedAdam(m.parameters()).copy_ema_to(dst)
