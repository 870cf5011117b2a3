"""Noise on every rollout step (`Fno2d.rollout(noise=...)`, `train_auto(noise_every_step=True)`) without a GPU: the host
restatement of the noise streams' counter mapping, the declarations of the new entry points, their argument checks
(all of which run before any device work) and the refusals of `Fno2d.rollout`, `add_input_noise` and `train_auto`.

`noise_stream_reference` is the host restatement the GPU tests compare the kernel against."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from cfdbench_b200 import RolloutNoise, _lib, add_input_noise, train_auto
from test_train_auto_host import _cpu_model, _Split
from test_train_noise_host import philox4x32_10, uniform_f32
from test_train_rollout_host import _TimedSplit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NEW_SYMBOLS = ["fno_add_input_noise_stream", "fno_rollout_noise", "fno_rollout_forward_train_noise",
               "fno_rollout_backward_noise", "fno_grid_rollout_noise", "fno_grid_rollout_forward_train_noise",
               "fno_grid_rollout_backward_noise"]


def stream_counter(q, j, step, stream):
    """The Philox counter of quad q of sample j at `step` in noise stream `stream`: (q + (stream << 16), j, step_lo,
    step_hi).  Stream 0 is fno_add_input_noise's counter."""
    q = np.asarray(q, np.uint64)
    ctr = np.zeros(q.shape + (4,), np.uint64)
    ctr[..., 0] = (q + (np.uint64(stream) << np.uint64(16))) & np.uint64(0xFFFFFFFF)
    ctr[..., 1] = j & 0xFFFFFFFF
    ctr[..., 2] = step & 0xFFFFFFFF
    ctr[..., 3] = step >> 32
    return ctr


def noise_stream_reference(seed: int, step: int, j: int, n_el: int, stream: int) -> np.ndarray:
    """The float64 normals z[0..n_el) of sample j at (seed, step) in noise stream `stream`: Box-Muller on the kernel's
    float32 uniforms, four normals per quad."""
    nq = (n_el + 3) // 4
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint64)
    u = uniform_f32(philox4x32_10(stream_counter(np.arange(nq), j, step, stream), key)).astype(np.float64)
    r0, t0 = np.sqrt(-2.0 * np.log(u[:, 0])), 2.0 * u[:, 1]
    r1, t1 = np.sqrt(-2.0 * np.log(u[:, 2])), 2.0 * u[:, 3]
    z = np.stack([r0 * np.cos(np.pi * t0), r0 * np.sin(np.pi * t0), r1 * np.cos(np.pi * t1), r1 * np.sin(np.pi * t1)], 1)
    return z.reshape(-1)[:n_el]


# ------------------------------------------------------------------------------------------------ the stream mapping
@pytest.mark.parametrize("counter,key,expect", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_stream_zero_reproduces_the_known_answers(counter, key, expect):
    ctr = stream_counter(counter[0], counter[1], counter[2] | (counter[3] << 32), 0)
    assert [int(v) for v in ctr] == list(counter)
    got = philox4x32_10(ctr[None], np.array([key], np.uint64))[0]
    assert [int(v) for v in got] == list(expect)


def test_streams_never_share_a_counter():
    q = np.arange(2 * 128 * 128 // 4)   # every quad of the largest frame
    words = [set(stream_counter(q, 5, 9, k)[:, 0].tolist()) for k in (0, 1, 2, 3, 255, 2 ** 16 - 1)]
    for a in range(len(words)):
        assert len(words[a]) == q.size
        for b in range(a):
            assert not words[a] & words[b], (a, b)
    # the other words do not depend on the stream
    assert np.array_equal(stream_counter(q, 5, 2 ** 40 + 9, 7)[:, 1:], stream_counter(q, 5, 2 ** 40 + 9, 0)[:, 1:])


def test_stream_reference():
    from test_train_noise_host import noise_reference
    n_el = 2 * 25 * 127   # odd H*W: the last quad is partial
    z0 = noise_stream_reference(2 ** 40 + 5, 7, 3, n_el, 0)
    assert np.array_equal(z0, noise_reference(2 ** 40 + 5, 7, 3, n_el))
    for k in (1, 2, 7, 2 ** 16 - 1):
        zk = noise_stream_reference(2 ** 40 + 5, 7, 3, n_el, k)
        assert np.all(np.isfinite(zk)) and not np.any(zk == z0), k
        assert abs(zk.mean()) < 6 / np.sqrt(n_el) and abs(zk.var() - 1) < 6 * np.sqrt(2 / n_el)


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


def test_new_entry_points_are_declared_and_exported(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read(), flags=re.S)
    raw = C.CDLL(_lib.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert re.search(rf"\bint\s+{name}\s*\(", hdr), name
        assert hasattr(raw, name) and name in _lib.SIGNATURES, name
    assert re.search(r"typedef struct fno_noise\b", hdr)
    assert [f for f, _ in _lib.FnoNoise._fields_] == ["std", "seed", "idx", "step_base", "step_offset", "k0"]
    assert lib.fno_version() == 4


def _err(lib) -> str:
    return lib.fno_last_error().decode()


def test_stream_entry_point_rejects_bad_arguments(lib):
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first

    def call(i=one, o=one, m=one, idx=one, n=4, h=64, w=64, std=1.0, seed=1, base=one, off=one, k=0):
        return lib.fno_add_input_noise_stream(i, o, m, idx, n, h, w, std, seed, base, off, k, C.c_void_p(0))
    for kw in (dict(i=None), dict(o=None), dict(m=None), dict(idx=None), dict(base=None), dict(n=0), dict(n=-1),
               dict(std=-1.0), dict(std=float("nan")), dict(std=float("inf")), dict(k=-1), dict(k=2 ** 16),
               dict(k=2 ** 31 - 1), dict(h=66, w=65, k=-5), dict(h=25, w=127, o=None)):
        assert call(**kw) == 1, kw
        assert "fno_add_input_noise_stream" in _err(lib)
    for h, w in ((23, 64), (64, 129), (0, 0)):
        assert call(h=h, w=w, k=-1) == 3
        assert "fno_add_input_noise_stream" in _err(lib)


def _noise(std=0.5, idx=16, base=16, k0=0):
    return _lib.FnoNoise(std, 3, idx, base, None, k0)


BAD_NOISE = [None, _noise(idx=None), _noise(base=None), _noise(std=-1.0), _noise(std=float("nan")),
             _noise(std=float("inf")), _noise(k0=-1), _noise(k0=2 ** 16 - 1), _noise(k0=2 ** 16)]   # the last two at 2 steps


def _structs():
    w, wb, sv, sc, ws = _lib.FnoWeights(), _lib.FnoWeightsBwd(), _lib.FnoTrainSaved(), _lib.FnoBwdScratch(), _lib.FnoWorkspace()
    w.n_layers, w.n_case_params = 4, 5
    fake = 4096   # never dereferenced
    sv.act[0] = fake
    sc.d[0] = sc.d[1] = sc.dz1 = sc.gm = sc.gwk = sc.partials = fake
    ws.ym = ws.z = fake
    return w, wb, sv, sc, ws


@pytest.mark.parametrize("grid", [False, True])
def test_noise_drivers_reject_bad_noise_before_device_work(lib, grid):
    """Every other argument is valid (fake addresses that are never dereferenced): a call that got as far as the
    device would fail with another status, so status 1 naming the entry point proves the noise check came first."""
    w, wb, sv, sc, ws = _structs()
    r, f = C.byref, 4096
    pre = "fno_grid_" if grid else "fno_"
    tail = (2, 66, 65, None) if grid else (2, 0, None)
    calls = {
        "rollout_noise": lambda nz, fed: getattr(lib, pre + "rollout_noise")(r(w), f, f, f, f, 2, r(ws), nz, fed, *tail),
        "rollout_forward_train_noise": lambda nz, fed: getattr(lib, pre + "rollout_forward_train_noise")(
            r(w), f, f, f, f, 2, r(sv), r(ws), nz, fed, *tail),
        "rollout_backward_noise": lambda nz, fed: getattr(lib, pre + "rollout_backward_noise")(
            r(w), r(wb), f, f, f, f, f, 2, r(sv), None, r(sc), r(ws), nz, fed, f + 4096, f + 8192, None, *tail),
    }
    for name, fn in calls.items():
        for nz in BAD_NOISE:
            assert fn(None if nz is None else r(nz), f) == 1, (name, nz and (nz.std, nz.idx, nz.step_base, nz.k0))
            assert pre + name in _err(lib) and "noise" in _err(lib), _err(lib)
        assert fn(r(_noise()), None) == 1   # no fed-frames buffer
        assert pre + name in _err(lib)
    if grid:   # the grid check comes first
        st = lib.fno_grid_rollout_noise(r(w), f, f, f, f, 2, r(ws), None, f, 2, 23, 65, None)
        assert st == 3 and "23x65" in _err(lib)


def _full_structs():
    """Structs with every buffer a driver checks set (fake addresses, never dereferenced)."""
    w, wb, sv, sc, ws = _structs()
    f = 4096
    ws.act[0] = ws.act[1] = ws.xm = f
    w.gx = w.gy = f
    for l in range(w.n_layers):
        sv.act[l + 1] = sv.pre[l] = sv.xm[l] = f
    return w, sv, ws


@pytest.mark.parametrize("grid", [False, True])
def test_noise_forward_drivers_check_the_forward_before_the_first_noise_launch(lib, grid):
    """With k0 >= 1 step 0's noise runs before step 0's forward: whatever the forward refuses must be refused first,
    with the forward's status and the entry point's name (status 1 for an argument, 3 for n_layers)."""
    r, f = C.byref, 4096
    nz = r(_noise(k0=1))
    pre = "fno_grid_" if grid else "fno_"

    def call(name, inputs=f, mask=f, cp=f, batch=2, act=0, edit=None):
        w, sv, ws = _full_structs()
        if edit:
            edit(w, sv, ws)
        tail = (batch, 66, 65, None) if grid else (batch, act, None)
        fn = getattr(lib, pre + name)
        if name == "rollout_noise":
            return fn(r(w), inputs, mask, cp, f, 2, r(ws), nz, f, *tail)
        return fn(r(w), inputs, mask, cp, f, 2, r(sv), r(ws), nz, f, *tail)
    cases = [dict(mask=None), dict(inputs=None), dict(batch=0), dict(batch=-1), dict(cp=None),
             dict(edit=lambda w, sv, ws: setattr(ws, "ym", None)),
             dict(edit=lambda w, sv, ws: setattr(ws, "z", None))]
    inference = [dict(edit=lambda w, sv, ws: ws.act.__setitem__(1, None)),
                 dict(edit=lambda w, sv, ws: setattr(ws, "xm", None))]
    training = [dict(edit=lambda w, sv, ws: sv.act.__setitem__(0, None)),
                dict(edit=lambda w, sv, ws: sv.pre.__setitem__(3, None))]
    extra = [dict(edit=lambda w, sv, ws: setattr(w, "gx", None))] if grid else [dict(act=2), dict(act=-1)]
    for name, own in (("rollout_noise", inference), ("rollout_forward_train_noise", training)):
        for kw in cases + own + extra:
            assert call(name, **kw) == 1, (name, kw)
            assert pre + name in _err(lib), (name, kw, _err(lib))
        for n_layers in (0, 9):
            assert call(name, edit=lambda w, sv, ws, n=n_layers: setattr(w, "n_layers", n)) == 3, (name, n_layers)
            assert pre + name in _err(lib)


# ------------------------------------------------------------------------------------------------ Python refusals
def _bad_records(b):
    ids = torch.zeros(b, dtype=torch.int64)
    return [
        ((0.1, 0, 1, ids, 0), None),   # a plain tuple, not a RolloutNoise
        (RolloutNoise(-1.0, 0, 1, ids, 0), "noise_std must be a real number >= 0"),
        (RolloutNoise(float("nan"), 0, 1, ids, 0), "noise_std must be a real number >= 0"),
        (RolloutNoise(0.1, -1, 1, ids, 0), r"noise_seed must be an int in \[0, 2\^64\)"),
        (RolloutNoise(0.1, 0, -1, ids, 0), r"noise_step must be an int in \[0, 2\^63\)"),
        (RolloutNoise(0.1, 0, 1.0, ids, 0), r"noise_step must be an int in \[0, 2\^63\)"),
        (RolloutNoise(0.1, 0, 1, ids.int(), 0), "noise.ids must be a"),
        (RolloutNoise(0.1, 0, 1, ids[:-1], 0), "noise.ids must be a"),
        (RolloutNoise(0.1, 0, 1, [0] * b, 0), "noise.ids must be a"),
        (RolloutNoise(0.1, 0, 1, ids, -1), "noise.k0 must be an int >= 0"),
        (RolloutNoise(0.1, 0, 1, ids, 1.0), "noise.k0 must be an int >= 0"),
        (RolloutNoise(0.1, 0, 1, ids, True), "noise.k0 must be an int >= 0"),
        (RolloutNoise(0.1, 0, 1, ids, 2 ** 16 - 2), r"k0 \+ steps <= 2\^16"),   # with steps = 3
    ]


def test_rollout_rejects_bad_noise_before_device_work():
    m = _cpu_model()
    b = 3
    x, cp, mk = torch.zeros(b, 2, 64, 64), torch.zeros(b, m.n_case_params), torch.ones(b, 64, 64)
    for noise, match in _bad_records(b):
        with pytest.raises(ValueError, match=match or "noise must be a RolloutNoise"):
            m.rollout(x, cp, mk, 3, noise=noise)
    ids = torch.zeros(b, dtype=torch.int64)
    # valid records (std 0 included, and the last stream) get as far as the CPU model's refusal
    for noise in (None, RolloutNoise(0.0, 0, 0, ids), RolloutNoise(0.5, 2 ** 64 - 1, 2 ** 63 - 1, ids, 2 ** 16 - 3),
                  RolloutNoise(np.float32(0.1), np.uint64(3), np.int64(2), ids, np.int32(1))):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            m.rollout(x, cp, mk, 3, noise=noise)


def test_add_input_noise_rejects_bad_arguments():
    b = 2
    fr, mk, ids = torch.zeros(b, 2, 64, 64), torch.ones(b, 1, 64, 64), torch.zeros(b, dtype=torch.int64)
    for kw, match in ((dict(std=-1.0), "std must be a real number >= 0"), (dict(seed=2 ** 64), "noise_seed"),
                      (dict(step=-1), "noise_step"), (dict(stream=-1), "stream must be an int"),
                      (dict(stream=2 ** 16), "stream must be an int"), (dict(stream=1.0), "stream must be an int"),
                      (dict(frames=fr[:, :1]), "frames must be"), (dict(frames=fr.double()), "frames must be"),
                      (dict(mask=mk[:1]), "mask must be"), (dict(ids=ids[:1]), "ids must be"),
                      (dict(ids=ids.int()), "ids must be"), (dict(), "CUDA device")):
        args = dict(frames=fr, mask=mk, ids=ids, std=0.1, seed=1, step=1, stream=1)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            add_input_noise(**args)


def test_train_auto_rejects_a_bad_noise_every_step(tmp_path):
    out = tmp_path / "out"
    tr, dv = _TimedSplit(12), _Split(3)
    m = _cpu_model()
    for v in (1, 0, "yes", None, np.bool_(True)):
        with pytest.raises(ValueError, match="noise_every_step must be a bool"):
            train_auto(m, tr, dv, out, rollout_steps=3, input_noise_std=0.1, noise_every_step=v)
    for kw in (dict(noise_every_step=True), dict(rollout_steps=3, noise_every_step=True),
               dict(rollout_steps=3, rollout_grad_steps=1, input_noise_std=0.1, noise_every_step=True),
               dict(rollout_steps=3, input_noise_std=0.1, noise_every_step=False)):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            train_auto(m, tr, dv, out, **kw)
    assert not out.exists()
