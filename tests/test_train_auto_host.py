"""`train_auto` (the graph-replayed replacement of the reference's `train_auto.train`, src/train_auto.py:181-313) without a
GPU: the new entry points' declarations and argument checks, the Adam coefficient table against the arithmetic of
`fno_adam_step`, the visiting order against a real DataLoader loop, and the argument checks of `train_auto`, all of
which run before any device work."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

import cfdbench_b200
from cfdbench_b200 import _lib, train_auto
from cfdbench_b200.loss import MseLoss
from cfdbench_b200.train import index_stream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("fno_train_stage_indices", "fno_adam_step_dev", "fno_adam_coefficients", "fno_train_log_step")


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
    assert lib.fno_version() == 4
    assert "train_auto" in cfdbench_b200.__all__


def test_new_entry_points_reject_bad_arguments(lib):
    st = C.c_void_p(0)
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first

    def stage(perm=one, n=10, stride=4, b=4, cur=one, out=one):
        return lib.fno_train_stage_indices(perm, n, stride, b, cur, out, st)
    for kw in (dict(perm=None), dict(cur=None), dict(out=None), dict(n=0), dict(stride=0), dict(b=0), dict(b=-1),
               dict(b=5), dict(n=3)):   # b > stride, b > n_perm
        assert stage(**kw) == 1, kw
        assert b"fno_train_stage_indices" in lib.fno_last_error()

    t = _lib.FnoAdamTensors()
    t.count = 1
    t.param[0] = t.grad[0] = t.exp_avg[0] = t.exp_avg_sq[0] = 16
    t.n[0] = 8

    def adam(tab=t, coef=one, n=4, cur=one):
        return lib.fno_adam_step_dev(C.byref(tab) if tab is not None else None, coef, n, cur, 0.9, 0.999, 1e-8, 0.0, st)
    for kw in (dict(tab=None), dict(coef=None), dict(cur=None), dict(n=0), dict(coef=C.c_void_p(20))):
        assert adam(**kw) == 1, kw
        assert b"fno_adam_step_dev" in lib.fno_last_error()
    bad = _lib.FnoAdamTensors.from_buffer_copy(t)
    bad.n[0] = 0
    assert adam(tab=bad) == 1
    bad = _lib.FnoAdamTensors.from_buffer_copy(t)
    bad.count = _lib.ADAM_MAX_TENSORS + 1
    assert adam(tab=bad) == 1
    bad = _lib.FnoAdamTensors.from_buffer_copy(t)
    bad.grad[0] = None
    assert adam(tab=bad) == 1

    def adam_host(tab=t, step=1):   # the host-coefficient form
        return lib.fno_adam_step(C.byref(tab) if tab is not None else None, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, st)
    for kw in (dict(tab=None), dict(step=0), dict(tab=bad)):
        assert adam_host(**kw) == 1, kw
        assert lib.fno_last_error().startswith(b"fno_adam_step:")

    out = (C.c_float * 8)()
    assert lib.fno_adam_coefficients(1e-3, 0.9, 0.999, 0, 4, out) == 1
    assert lib.fno_adam_coefficients(1e-3, 0.9, 0.999, 1, 0, out) == 1
    assert lib.fno_adam_coefficients(1e-3, 0.9, 0.999, 1, 4, None) == 1
    assert b"fno_adam_coefficients" in lib.fno_last_error()

    for args in ((None, one, 4, one), (one, None, 4, one), (one, one, 0, one), (one, one, 4, None)):
        assert lib.fno_train_log_step(*args, st) == 1
        assert b"fno_train_log_step" in lib.fno_last_error()


@pytest.mark.parametrize("lr", [1e-3, 3e-4, 0.1, 1e-3 * 0.9 ** 37, 7.5e-6])
def test_adam_coefficients_match_fno_adam_step_arithmetic(lib, lr):
    """The table equals, bit for bit, what launch_adam_step passes the kernel: lr, beta1, beta2 as float32, pow in
    double, then a float32 cast (torch.optim.Adam's _single_tensor_adam forms them the same way)."""
    n = 100_000
    out = np.empty((n, 2), np.float32)
    b1, b2 = 0.9, 0.999
    assert lib.fno_adam_coefficients(lr, b1, b2, 1, n, out.ctypes.data) == 0
    lr32, b1_32, b2_32 = (float(np.float32(v)) for v in (lr, b1, b2))
    steps = np.arange(1, n + 1)
    ref = np.empty_like(out)
    for i, s in enumerate(steps):
        bc1 = 1.0 - math.pow(b1_32, float(s))
        bc2 = 1.0 - math.pow(b2_32, float(s))
        ref[i, 0] = np.float32(lr32 / bc1)
        ref[i, 1] = np.float32(1.0 / math.sqrt(bc2))
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    # a table that starts later is the matching slice
    tail = np.empty((1000, 2), np.float32)
    assert lib.fno_adam_coefficients(lr, b1, b2, 5001, 1000, tail.ctypes.data) == 0
    assert np.array_equal(tail.view(np.uint32), out[5000:6000].view(np.uint32))


# ------------------------------------------------------------------------------------------------ visiting order
class _Indices(torch.utils.data.Dataset):
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return i


def _real_loop(n, batch_size, num_epochs, eval_interval, generator):
    """The reference's loop over a stand-in dataset: a DataLoader(shuffle=True) pass per epoch and, every eval_interval
    epochs, a pass of evaluate's DataLoader(shuffle=False)."""
    ds = _Indices(n)
    orders = []
    for ep in range(num_epochs):
        loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=True, generator=generator)
        orders.append(np.concatenate([b.numpy() for b in loader]).astype(np.int64))
        if (ep + 1) % eval_interval == 0:
            for _ in torch.utils.data.DataLoader(ds, batch_size=2, shuffle=False, generator=generator):
                pass
    return orders


@pytest.mark.parametrize("n,batch_size", [(37, 8), (32, 8), (5, 8), (9, 1), (1, 1), (100, 64)])
@pytest.mark.parametrize("eval_interval", [1, 2, 5])
@pytest.mark.parametrize("explicit", [False, True])
def test_index_stream_matches_dataloader_loop(n, batch_size, eval_interval, explicit):
    epochs = 6
    if explicit:
        ref = _real_loop(n, batch_size, epochs, eval_interval, torch.Generator().manual_seed(123))
        g = torch.Generator().manual_seed(123)
        got = index_stream(n, batch_size, epochs, eval_interval, g)
        after_ref = torch.randint(0, 2 ** 31, (4,), generator=_advance(123, n, batch_size, epochs, eval_interval))
        after_got = torch.randint(0, 2 ** 31, (4,), generator=g)
    else:
        torch.manual_seed(77)
        ref = _real_loop(n, batch_size, epochs, eval_interval, None)
        after_ref = torch.randint(0, 2 ** 31, (4,))
        torch.manual_seed(77)
        got = index_stream(n, batch_size, epochs, eval_interval, None)
        after_got = torch.randint(0, 2 ** 31, (4,))
    assert len(got) == epochs
    for a, b in zip(got, ref):
        assert a.dtype == np.int64 and np.array_equal(a, b)
        assert sorted(a.tolist()) == list(range(n))
    assert len({tuple(a.tolist()) for a in got}) > 1 or n <= 2
    assert torch.equal(after_ref, after_got)   # the RNG is left where the loop leaves it


def _advance(seed, n, batch_size, epochs, eval_interval):
    g = torch.Generator().manual_seed(seed)
    _real_loop(n, batch_size, epochs, eval_interval, g)
    return g


def test_device_frames_loader_order_is_unchanged():
    """DeviceFrames.loader's index stream (now index_batches) still equals a DataLoader's, batch by batch."""
    from cfdbench_b200.data import index_batches
    for shuffle in (False, True):
        for drop_last in (False, True):
            g1, g2 = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
            ref = [b.tolist() for b in torch.utils.data.DataLoader(_Indices(23), batch_size=4, shuffle=shuffle,
                                                                    generator=g1, drop_last=drop_last)]
            assert [list(b) for b in index_batches(23, 4, shuffle, g2, drop_last)] == ref
            assert torch.equal(torch.rand(3, generator=g1), torch.rand(3, generator=g2))


# ------------------------------------------------------------------------------------------------ train_auto checks
class _Split:
    def __init__(self, n, gh=64, gw=64, p=5):
        self.inputs = torch.zeros(n, 3, gh, gw)
        self.labels = torch.zeros(n, 3, gh, gw)
        self.case_ids = np.zeros(n, np.int64)
        self.case_params = [{f"p{j}": 0.0 for j in range(p)}]


def _cpu_model(loss="nmse", act_dtype="float32"):
    from cfdbench_b200 import Fno2d
    loss_fn = MseLoss(normalize=(loss == "nmse"))
    return Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_fn, num_layers=2, hidden_dim=32, modes1=12,
                 modes2=12, act_dtype=act_dtype, device="cpu")


def test_train_auto_rejects_bad_arguments(tmp_path):
    out = tmp_path / "out"
    tr, dv = _Split(4), _Split(3)
    m = _cpu_model()
    with pytest.raises(TypeError, match="Fno2d"):
        train_auto(torch.nn.Linear(2, 2), tr, dv, out)
    with pytest.raises(ValueError, match="nmse"):
        train_auto(_cpu_model(loss="mse"), tr, dv, out)
    for kw in (dict(num_epochs=0), dict(lr_step_size=0), dict(batch_size=0), dict(batch_size=-3), dict(eval_batch_size=0),
               dict(log_interval=0), dict(eval_interval=0), dict(batch_size=2.0), dict(num_epochs=True)):
        with pytest.raises(ValueError, match="positive int"):
            train_auto(m, tr, dv, out, **kw)
    with pytest.raises(ValueError, match="train_data is empty"):
        train_auto(m, _Split(0), dv, out)
    with pytest.raises(ValueError, match="dev_data is empty"):
        train_auto(m, tr, _Split(0), out)
    with pytest.raises(ValueError, match="dev_data must be"):
        train_auto(m, tr, object(), out)
    with pytest.raises(ValueError, match="supports"):
        train_auto(m, _Split(4, 20, 64), dv, out)   # the model's own grid check
    with pytest.raises(ValueError, match="act_dtype"):
        train_auto(_cpu_model(act_dtype="bfloat16"), _Split(4, 66, 65), _Split(3, 66, 65), out)
    for bad_tr, bad_dv, what in ((_Split(4, p=3), dv, "train_data"), (tr, _Split(3, p=6), "dev_data"),
                                 (_Split(4, 66, 65, p=0), _Split(3, 66, 65), "train_data")):
        with pytest.raises(ValueError, match=f"{what} has .* case parameters per sample, the model takes n_case_params=5"):
            train_auto(m, bad_tr, bad_dv, out)   # the captured forward would read past / misread the case parameters
    short = _Split(4)
    short.case_ids = short.case_ids[:3]
    with pytest.raises(ValueError, match="case_ids"):
        train_auto(m, short, dv, out)
    m16 = _cpu_model(act_dtype="bfloat16")
    m16.generic_grid_at_64 = True   # the grid path is fp32 only: refused by the model's own routing check
    with pytest.raises(ValueError, match="generic_grid_at_64"):
        train_auto(m16, tr, dv, out)
    frozen = _cpu_model()
    for prm in frozen.parameters():
        prm.requires_grad_(False)
    with pytest.raises(ValueError, match="frozen"):
        train_auto(frozen, tr, dv, out)
    m._dp_enabled = True
    with pytest.raises(ValueError, match="data parallel"):
        train_auto(m, tr, dv, out)
    m._dp_enabled = False
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, dv, out)
    assert not out.exists()   # rejected before anything was written
