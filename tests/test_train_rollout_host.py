"""Training through K-step rollouts (`train_auto(rollout_steps=K)`) without a GPU: the new entry points' declarations
and argument checks, `rollout_windows` against a brute-force enumeration, the window visiting order against a real
DataLoader loop, and the argument checks of `train_auto`, all of which run before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import cfdbench_b200
from cfdbench_b200 import _lib, rollout_windows, train_auto
from cfdbench_b200.train import epoch_permutation
from test_train_auto_host import _cpu_model, _Split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("fno_gather_window", "fno_grid_gather_window", "fno_loss_seq_fwd", "fno_loss_seq_bwd")


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
    assert re.search(r"\bsize_t\s+fno_loss_seq_scratch_bytes\s*\(", hdr)
    assert lib.fno_version() == 4
    assert "rollout_windows" in cfdbench_b200.__all__ and "train_auto" in cfdbench_b200.__all__


def test_loss_seq_scratch_bytes(lib):
    one = lib.fno_loss_scratch_bytes()
    for k in (1, 2, 8, 100):
        assert lib.fno_loss_seq_scratch_bytes(k) >= k * (one - 16) + 4 * (k + 1)
    assert lib.fno_loss_seq_scratch_bytes(0) == 0 and lib.fno_loss_seq_scratch_bytes(-1) == 0


def test_new_entry_points_reject_bad_arguments(lib):
    st = C.c_void_p(0)
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first

    def gather(grid=False, fin=one, fout=one, table=one, ids=one, idx=one, n_idx=4, p=5, dtype=_lib.ACT_F32, inputs=one,
               label=one, mask=one, cp=one, steps=3, s=1, n_frames=10, seq=one, h=66, w=65):
        args = (fin, fout, table, ids, idx, n_idx, p, dtype, inputs, label, mask, cp, steps, s, n_frames, seq)
        if grid:
            return lib.fno_grid_gather_window(*args, h, w, st)
        return lib.fno_gather_window(*args, st)
    for grid in (False, True):
        name = b"fno_grid_gather_window" if grid else b"fno_gather_window"
        for kw in (dict(fin=None), dict(fout=None), dict(ids=None), dict(idx=None), dict(inputs=None), dict(mask=None),
                   dict(seq=None), dict(table=None), dict(cp=None), dict(n_idx=0), dict(n_idx=-2), dict(p=-1),
                   dict(p=17), dict(dtype=7), dict(steps=0), dict(steps=-1), dict(steps=40000), dict(s=0), dict(s=-2),
                   dict(n_frames=0)):
            assert gather(grid, **kw) == 1, (grid, kw)
            assert name in lib.fno_last_error()
    for h, w in ((23, 64), (66, 129), (0, 0)):
        assert gather(True, h=h, w=w) == 3
        assert gather(True, h=h, w=w, steps=0) == 3   # the grid check comes first

    def fwd(preds=one, labels=one, n=100, steps=2, scratch=one, out=one):
        return lib.fno_loss_seq_fwd(preds, labels, n, steps, scratch, out, st)
    for kw in (dict(preds=None), dict(labels=None), dict(scratch=None), dict(out=None), dict(n=0), dict(steps=0),
               dict(steps=-3), dict(steps=40000)):
        assert fwd(**kw) == 1, kw
        assert b"fno_loss_seq_fwd" in lib.fno_last_error()

    def bwd(preds=one, labels=one, f=one, g=one, d=one, n=100, steps=2):
        return lib.fno_loss_seq_bwd(preds, labels, f, g, d, n, steps, st)
    for kw in (dict(preds=None), dict(labels=None), dict(f=None), dict(g=None), dict(d=None), dict(n=0), dict(steps=0),
               dict(steps=-1)):
        assert bwd(**kw) == 1, kw
        assert b"fno_loss_seq_bwd" in lib.fno_last_error()


# ------------------------------------------------------------------------------------------------ windows
def _brute(case_ids, steps, s):
    n = len(case_ids)
    out = []
    for j in range(n):
        ks = [j + k * s for k in range(steps)]
        if ks[-1] < n and all(case_ids[i] == case_ids[j] for i in ks):
            out.append(j)
    return out


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("s", [1, 2, 5])
def test_rollout_windows_match_brute_force(seed, s):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, 25, size=rng.integers(1, 7))
    case_ids = np.repeat(np.arange(len(lengths)), lengths)
    for steps in range(1, 7):
        got = rollout_windows(case_ids, steps, s)
        assert got.dtype == np.int64
        assert got.tolist() == _brute(case_ids, steps, s), (lengths, steps)
    assert np.array_equal(rollout_windows(case_ids, 1, s), np.arange(len(case_ids)))
    assert np.array_equal(rollout_windows(list(case_ids), 3, s), rollout_windows(case_ids, 3, s))


def test_rollout_windows_rejects_bad_arguments():
    assert rollout_windows([0, 0, 1], 4, 1).size == 0
    assert rollout_windows([], 1, 1).size == 0
    for steps, s in ((0, 1), (1, 0), (-1, 1), (2.0, 1), (True, 1), (2, None)):
        with pytest.raises(ValueError, match="positive int"):
            rollout_windows([0, 0, 0], steps, s)


class _Indices(torch.utils.data.Dataset):
    def __init__(self, values):
        self.values = values

    def __len__(self):
        return len(self.values)

    def __getitem__(self, i):
        return int(self.values[i])


@pytest.mark.parametrize("explicit", [False, True])
@pytest.mark.parametrize("batch_size", [1, 4, 64])
def test_window_order_matches_dataloader_over_the_windows(explicit, batch_size):
    """Each epoch visits what a DataLoader(shuffle=True) over the |V| windows visits, drawing the same RNG."""
    case_ids = np.repeat(np.arange(4), [9, 3, 12, 7])
    windows = rollout_windows(case_ids, 4, 2)
    assert 0 < windows.size < case_ids.size
    ds = _Indices(windows)
    for _ in range(2 if explicit else 1):
        g_ref, g = (torch.Generator().manual_seed(11), torch.Generator().manual_seed(11)) if explicit else (None, None)
        if not explicit:
            torch.manual_seed(11)
        ref = [np.concatenate([b.numpy() for b in torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=True,
                                                                              generator=g_ref)]) for _ in range(3)]
        after_ref = torch.randint(0, 2 ** 31, (4,), generator=g_ref)
        if not explicit:
            torch.manual_seed(11)
        got = [windows[epoch_permutation(windows.size, batch_size, g)] for _ in range(3)]
        after = torch.randint(0, 2 ** 31, (4,), generator=g)
        for a, b in zip(got, ref):
            assert np.array_equal(a, b) and sorted(a.tolist()) == windows.tolist()
        assert torch.equal(after, after_ref)


# ------------------------------------------------------------------------------------------------ train_auto checks
class _TimedSplit(_Split):
    def __init__(self, n, s=1, n_cases=2, **kw):
        super().__init__(n, **kw)
        self.case_ids = np.repeat(np.arange(n_cases), [n // n_cases] * (n_cases - 1) + [n - n // n_cases * (n_cases - 1)])
        self.case_params = [{f"p{j}": 0.0 for j in range(5)} for _ in range(n_cases)]
        self.time_step_size = s


def test_train_auto_rejects_bad_rollout_arguments(tmp_path):
    out = tmp_path / "out"
    tr, dv = _TimedSplit(12), _Split(3)
    m = _cpu_model()
    for k in (0, -1, 2.0, True, "2"):
        with pytest.raises(ValueError, match="rollout_steps must be a positive int"):
            train_auto(m, tr, dv, out, rollout_steps=k)
    for s in (0, -2, 1.5):
        with pytest.raises(ValueError, match="time_step_size must be a positive int"):
            train_auto(m, tr, dv, out, rollout_steps=2, time_step_size=s)
        with pytest.raises(ValueError, match="time_step_size must be a positive int"):
            train_auto(m, tr, dv, out, time_step_size=s)
    with pytest.raises(ValueError, match="needs a time_step_size"):
        train_auto(m, _Split(12), dv, out, rollout_steps=2)   # the dataset has no time_step_size
    bad = _TimedSplit(12, s=0)
    with pytest.raises(ValueError, match="time_step_size must be a positive int"):
        train_auto(m, bad, dv, out, rollout_steps=2)
    with pytest.raises(ValueError, match="no 7-step window"):
        train_auto(m, tr, dv, out, rollout_steps=7)   # cases of 6 samples
    with pytest.raises(ValueError, match="no 3-step window"):
        train_auto(m, tr, dv, out, rollout_steps=3, time_step_size=3)
    # a valid rollout set-up gets as far as the CPU model's refusal
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, dv, out, rollout_steps=6)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, _Split(12), dv, out, rollout_steps=2, time_step_size=1)
    assert not out.exists()   # rejected before anything was written
