"""Teacher forcing of a rollout (scheduled sampling: `Fno2d.rollout(teacher=...)`, `train_auto(teacher_forcing=...)`)
without a GPU: the host restatement of the flag draw, the declarations of the new entry points, their argument and
alignment checks (all before any device work), the refusals of `Fno2d.rollout`, `teacher_forcing_flags` and
`train_auto`, the resume record, and the float64 oracle of the teacher-forced rollout's backward.

`teacher_flags_reference` and `teacher_rollout_vjp` are the yardsticks the GPU tests compare against."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import cfdbench_b200
from cfdbench_b200 import TeacherForcing, _lib, resume, synth, teacher_forcing_flags, train_auto
from oracle.fno_numpy import _scipy_erf, fno_forward, fno_vjp, fno_vjp_saved
from oracle.fno_rollout_numpy import fno_rollout_vjp
from test_train_auto_host import _cpu_model, _Split
from test_train_noise_host import philox4x32_10, uniform_f32
from test_train_resume_host import DEFAULTS, _state
from test_train_rollout_host import _TimedSplit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["fno_teacher_flags", "fno_rollout_forward_train_feed", "fno_rollout_backward_feed",
               "fno_grid_rollout_forward_train_feed", "fno_grid_rollout_backward_feed"]


# ------------------------------------------------------------------------------------------------ the flag draw
def teacher_words(seed: int, step: int, ids, steps: int) -> np.ndarray:
    """(steps - 1, B) uint32: word x0 of Philox4x32-10(counter = (s, j, step_lo, step_hi), key = (seed_lo, seed_hi)) for
    rollout steps s = 1 .. steps - 1 and j = ids[b]."""
    ids = np.asarray(ids, dtype=np.int64)
    ctr = np.zeros((steps - 1, ids.size, 4), np.uint64)
    ctr[..., 0] = np.arange(1, steps)[:, None]
    ctr[..., 1] = (ids.astype(np.uint64) & np.uint64(0xFFFFFFFF))[None, :]
    ctr[..., 2] = step & 0xFFFFFFFF
    ctr[..., 3] = step >> 32
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint64)
    return philox4x32_10(ctr, key)[..., 0]


def teacher_flags_reference(seed: int, step: int, ids, steps: int, prob: float) -> np.ndarray:
    """The (steps - 1, B) uint8 flags of fno_teacher_flags: uniform_f32(word) <= prob in float32."""
    return (uniform_f32(teacher_words(seed, step, ids, steps)) <= np.float32(prob)).astype(np.uint8)


@pytest.mark.parametrize("seed,step,ids,steps,words,flags_half", [
    (0, 1, [0, 1, 2], 3, [[0xCA7CF69E, 0x8DE34A00, 0x040D2697], [0xC5FA1393, 0xC37FFB06, 0x6DE2493F]],
     [[0, 0, 1], [0, 0, 1]]),
    (2 ** 63 + 9, 2 ** 40 + 3, [7, 123456789], 4, [[0xC61261E9, 0x1E6E0E37], [0xAF51DF19, 0xD9050118],
                                                   [0xCEC9B691, 0xBF4CC538]], [[0, 1], [0, 0], [0, 0]]),
])
def test_flag_reference_reproduces_the_known_answers(seed, step, ids, steps, words, flags_half):
    assert teacher_words(seed, step, ids, steps).tolist() == words
    assert teacher_flags_reference(seed, step, ids, steps, 0.5).tolist() == flags_half


def test_prob_zero_sets_no_flag_and_prob_one_every_flag():
    ids = np.arange(4000) * 7919
    assert teacher_flags_reference(3, 11, ids, 5, 0.0).sum() == 0
    assert teacher_flags_reference(3, 11, ids, 5, 1.0).all()
    # the extreme words: u = 2^-33 > 0 and u rounds to exactly 1
    assert uniform_f32(np.uint32(0)) > 0 and uniform_f32(np.uint32(0xFFFFFFFF)) == np.float32(1.0)


def test_flags_depend_on_the_sample_not_the_slot_and_hit_the_rate():
    ids = np.arange(20000) + 5
    f = teacher_flags_reference(9, 4, ids, 3, 0.3)
    perm = np.random.default_rng(0).permutation(ids.size)
    assert np.array_equal(teacher_flags_reference(9, 4, ids[perm], 3, 0.3), f[:, perm])
    n = f.size
    assert abs(f.mean() - 0.3) <= 4 * np.sqrt(0.3 * 0.7 / n)
    assert not np.array_equal(f, teacher_flags_reference(10, 4, ids, 3, 0.3))   # the seed matters
    assert not np.array_equal(f, teacher_flags_reference(9, 5, ids, 3, 0.3))    # and the step


# ------------------------------------------------------------------------------------------------ the float64 oracle
def teacher_rollout_vjp(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray, gpreds_seq: np.ndarray,
                        teacher: np.ndarray, flags: np.ndarray, frames=None, erf=_scipy_erf):
    """`oracle.fno_rollout_numpy.fno_rollout_vjp` for a teacher-forced rollout: step s >= 1 of sample b is fed
    teacher[s-1][b] where flags[s-1][b] is set, else preds_{s-1}[b] -- this oracle's own float64 prediction, or
    frames[s-1][b] when `frames` is given (the GPU's trajectory, as fno_rollout_vjp's `frames`).  The sweep hands a
    forced sample's prediction s - 1 the upstream gradient gpreds_seq[s-1] alone (no carry), every other sample's
    gpreds_seq[s-1] + dL/d(frame fed to step s).  Returns (parameter gradients, dL/dinputs, dL/dcase_params)."""
    steps = len(gpreds_seq)
    m = (mask[:, None] if mask.ndim == 3 else mask).astype(np.float64)
    x = [np.asarray(inputs, dtype=np.float64)]
    for s in range(1, steps):
        pred = fno_forward(sd, x[-1], case_params, m)["preds"] if frames is None else np.asarray(frames[s - 1], np.float64)
        forced = np.asarray(flags[s - 1], bool)[:, None, None, None]
        x.append(np.where(forced, np.asarray(teacher[s - 1], np.float64), pred))
    grads: dict = {}
    d_cp = carry = None
    for s in reversed(range(steps)):
        fwd = fno_forward(sd, x[s], case_params, m, return_acts=True)
        up = np.asarray(gpreds_seq[s], dtype=np.float64)
        if carry is not None:
            up = up + carry
        g, dx, dcp_s = fno_vjp_saved(sd, x[s], case_params, m, up, fwd["acts"], fwd["pres"], erf=erf)
        for k, v in g.items():
            grads[k] = v if k not in grads else grads[k] + v
        d_cp = dcp_s if d_cp is None else d_cp + dcp_s
        carry = dx if s == 0 else np.where(np.asarray(flags[s - 1], bool)[:, None, None, None], 0.0, dx)
    return grads, carry, d_cp


def _case(seed, b, gh, gw, p, depth, steps):
    rng = np.random.default_rng(seed)
    sd = synth.make_state_dict(seed, n_params=p, depth=depth, spectral_gain=50.0)
    mask = np.ones((b, 1, gh, gw))
    mask[:, :, 0, :] = mask[:, :, :, gw - 1] = 0.0
    inputs = rng.standard_normal((b, 2, gh, gw))
    cp = rng.standard_normal((b, p))
    gseq = rng.standard_normal((steps, b, 2, gh, gw))
    teacher = rng.standard_normal((steps - 1, b, 2, gh, gw)) * mask
    return sd, inputs, cp, mask, gseq, teacher


@pytest.mark.parametrize("grid", [(64, 64), (66, 65)], ids=["64x64", "66x65"])
def test_oracle_without_flags_is_the_rollout_vjp(grid):
    sd, inputs, cp, mask, gseq, teacher = _case(3, 2, *grid, 5, 2, 3)
    a = fno_rollout_vjp(sd, inputs, cp, mask, gseq)
    b = teacher_rollout_vjp(sd, inputs, cp, mask, gseq, teacher, np.zeros((2, 2), np.uint8))
    for k in a[0]:
        np.testing.assert_array_equal(a[0][k], b[0][k], err_msg=k)
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[2], b[2])


@pytest.mark.parametrize("grid", [(64, 64), (66, 65)], ids=["64x64", "66x65"])
def test_oracle_with_every_flag_is_the_sum_of_single_step_vjps(grid):
    steps = 3
    sd, inputs, cp, mask, gseq, teacher = _case(4, 2, *grid, 5, 2, steps)
    g, d_in, d_cp = teacher_rollout_vjp(sd, inputs, cp, mask, gseq, teacher, np.ones((steps - 1, 2), np.uint8))
    xs = [inputs] + [teacher[s] for s in range(steps - 1)]
    parts = [fno_vjp(sd, xs[s], cp, mask, gseq[s]) for s in range(steps)]
    for k in g:
        np.testing.assert_allclose(g[k], sum(p[0][k] for p in parts), rtol=1e-12, atol=1e-14, err_msg=k)
    np.testing.assert_array_equal(d_in, parts[0][1])
    np.testing.assert_allclose(d_cp, sum(p[2] for p in parts), rtol=1e-12, atol=1e-14)


def test_oracle_mixed_flags_cut_exactly_the_forced_carry():
    """Sample 0 forced at step 1, sample 1 never: d_inputs of sample 0 is step 0's own VJP, sample 1's is the chain's."""
    steps = 2
    sd, inputs, cp, mask, gseq, teacher = _case(5, 2, 64, 64, 5, 2, steps)
    flags = np.array([[1, 0]], np.uint8)
    _, d_in, _ = teacher_rollout_vjp(sd, inputs, cp, mask, gseq, teacher, flags)
    own = fno_vjp(sd, inputs, cp, mask, gseq[0])[1]
    chain = fno_rollout_vjp(sd, inputs, cp, mask, gseq)[1]
    np.testing.assert_array_equal(d_in[0], own[0])
    np.testing.assert_allclose(d_in[1], chain[1], rtol=1e-12, atol=1e-14)


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


def _err(lib) -> str:
    return lib.fno_last_error().decode()


def test_new_entry_points_are_declared_exported_and_public(lib):
    hdr = open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES and hasattr(lib, name), name
    assert "typedef struct fno_teacher" in hdr
    assert C.sizeof(_lib.FnoTeacher) == 2 * C.sizeof(C.c_void_p)
    assert lib.fno_version() == 4
    for name in ("TeacherForcing", "teacher_forcing_flags"):
        assert name in cfdbench_b200.__all__ and getattr(cfdbench_b200, name) is not None


def test_flag_entry_point_rejects_bad_arguments(lib):
    f = 4096   # never dereferenced

    def call(idx=f, batch=2, steps=3, prob=f, seed=1, base=f, off=None, flags=f):
        return lib.fno_teacher_flags(idx, batch, steps, prob, seed, base, off, flags, None)
    for kw in (dict(idx=None), dict(prob=None), dict(base=None), dict(flags=None), dict(batch=0), dict(batch=-1),
               dict(steps=1), dict(steps=0), dict(steps=2 ** 16 + 1), dict(steps=2 ** 16, batch=2 ** 16)):
        assert call(**kw) == 1, kw
        assert "fno_teacher_flags" in _err(lib)


def _structs():
    w, wb, sv, sc, ws = _lib.FnoWeights(), _lib.FnoWeightsBwd(), _lib.FnoTrainSaved(), _lib.FnoBwdScratch(), _lib.FnoWorkspace()
    w.n_layers, w.n_case_params = 4, 5
    fake = 4096
    sv.act[0] = fake
    for l in range(4):
        sv.act[l + 1] = sv.pre[l] = sv.xm[l] = fake
    sc.d[0] = sc.d[1] = sc.dz1 = sc.gm = sc.gwk = sc.partials = fake
    ws.ym = ws.z = ws.act[0] = ws.act[1] = ws.xm = fake
    w.gx = w.gy = fake
    return w, wb, sv, sc, ws


@pytest.mark.parametrize("grid", [False, True])
def test_feed_drivers_reject_a_bad_teacher_or_noise_before_device_work(lib, grid):
    w, wb, sv, sc, ws = _structs()
    r, f = C.byref, 4096
    pre = "fno_grid_" if grid else "fno_"
    tail = (2, 66, 65, None) if grid else (2, 0, None)
    fwd = lambda nz, tc, fed: getattr(lib, pre + "rollout_forward_train_feed")(r(w), f, f, f, f, 3, r(sv), r(ws), nz, tc,
                                                                             fed, *tail)
    bwd = lambda nz, tc, fed: getattr(lib, pre + "rollout_backward_feed")(r(w), r(wb), f, f, f, f, f, 3, r(sv), None,
                                                                        r(sc), r(ws), nz, tc, fed, f + 4096, f + 8192,
                                                                        None, *tail)
    bad_noise = _lib.FnoNoise(-1.0, 3, f, f, None, 0)
    for name, fn, need_frames in (("rollout_forward_train_feed", fwd, True), ("rollout_backward_feed", bwd, False)):
        for tc, fed in ((None, f), (_lib.FnoTeacher(f, None), f), (_lib.FnoTeacher(f, f), None)) + \
                ((_lib.FnoTeacher(None, f), f),) * need_frames:
            assert fn(None, None if tc is None else r(tc), fed) == 1, (name, tc and (tc.frames, tc.flags), fed)
            assert pre + name in _err(lib) and "teacher" in _err(lib), _err(lib)
        assert fn(r(bad_noise), r(_lib.FnoTeacher(f, f)), f) == 1
        assert pre + name in _err(lib) and "noise" in _err(lib), _err(lib)
    if grid:   # the grid check comes first
        st = lib.fno_grid_rollout_forward_train_feed(r(w), f, f, f, f, 3, r(sv), r(ws), None, None, f, 2, 23, 65, None)
        assert st == 3 and "23x65" in _err(lib)


# The alignment contract of the new entry points (the widest access their kernels make through each pointer), checked
# with the refusal machinery of test_abi_alignment_host in a child process that sees no CUDA device.
_HOST = "host / struct"
_TRAIN = dict(w=_HOST, saved=_HOST, ws=_HOST, noise=_HOST, teacher=_HOST, stream=_HOST)
_BWD = dict(w=_HOST, wb=_HOST, saved=_HOST, grads=_HOST, scratch=_HOST, ws=_HOST, noise=_HOST, teacher=_HOST,
            stream=_HOST)
TEACHER_ALIGN = {
    "fno_teacher_flags": dict(idx=8, prob=4, step_base=8, step_offset=4, flags=1, stream=_HOST),   # flags: bytes
    "fno_rollout_forward_train_feed": dict(_TRAIN, inputs=16, mask=16, case_params=4, preds_seq=16, fed=16),
    "fno_rollout_backward_feed": dict(_BWD, inputs=16, mask=16, case_params=4, preds_seq=16, dpreds_seq=16, fed=16,
                                      carry=16, d_inputs=16, d_case_params=4),
    "fno_grid_rollout_forward_train_feed": dict(_TRAIN, inputs=4, mask=4, case_params=4, preds_seq=4, fed=4),
    "fno_grid_rollout_backward_feed": dict(_BWD, inputs=4, mask=4, case_params=4, preds_seq=4, dpreds_seq=4, fed=4,
                                           carry=4, d_inputs=4, d_case_params=4),
}

_CHILD = """
import json, re, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_abi_alignment_host as t
from test_teacher_forcing_host import TEACHER_ALIGN
from cfdbench_b200 import _lib as L
t.ALIGN.update(TEACHER_ALIGN)   # this child process only
structs = t._structs
def with_teacher(lib_mod, fake, grid):
    st = structs(lib_mod, fake, grid)
    st["teacher"] = L.FnoTeacher(fake(), fake())
    return st
t._structs = with_teacher
lib = L.load()
src = re.sub(r"/\\*.*?\\*/", "", open(t.HEADER).read(), flags=re.S)
decls = {{m.group(1): m.group(2) for m in re.finditer(r"\\bfno_status\\s+(fno_\\w+)\\s*\\(([^)]*)\\)\\s*;", src)}}
rows = []
for name, table in TEACHER_ALIGN.items():
    for target, need in table.items():
        if need == t.HOST:
            continue
        for offset in (1, 2, 4, 8):
            if offset >= need:
                continue
            args, keep = t._args(name, decls[name], L, t._Fake(), 0, target, offset)
            status = getattr(lib, name)(*args)
            rows.append((name, target, 0, offset, need, status, lib.fno_last_error().decode()))
print("ROWS" + json.dumps(rows))
"""


def test_new_entry_points_refuse_under_aligned_pointers_before_device_work(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read(), flags=re.S)
    for name, table in TEACHER_ALIGN.items():   # the table names every pointer parameter
        params = re.search(rf"\b{name}\s*\(([^)]*)\)", hdr).group(1)
        ptrs = {re.findall(r"\w+", p)[-1] for p in params.split(",") if "*" in p}
        assert ptrs == set(table), (name, ptrs ^ set(table))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    rows = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("ROWS")][-1][4:])
    assert len(rows) >= 40
    bad = [row for row in rows if not (row[5] == 1 and row[6] == f"{row[0]}: {row[1]} must be {row[4]}-byte aligned")]
    assert not bad, "\n".join(map(str, bad))


# ------------------------------------------------------------------------------------------------ Python refusals
def test_rollout_rejects_a_bad_teacher_before_device_work():
    m = _cpu_model()
    b, K = 3, 3
    x, cp, mk = torch.zeros(b, 2, 64, 64), torch.zeros(b, m.n_case_params), torch.ones(b, 64, 64)
    fr, fl = torch.zeros(K - 1, b, 2, 64, 64), torch.zeros(K - 1, b, dtype=torch.uint8)
    for teacher, match in (((fr, fl), "teacher must be a TeacherForcing"),
                           (TeacherForcing(fr[:1], fl), "teacher.frames must be"),
                           (TeacherForcing(fr.double(), fl), "teacher.frames must be"),
                           (TeacherForcing(fr[:, :, :, :63], fl), "teacher.frames must be"),
                           (TeacherForcing(fr.clone().requires_grad_(True), fl), "requires grad"),
                           (TeacherForcing(fr, fl[:, :2]), "teacher.flags must be"),
                           (TeacherForcing(fr, fl.int()), "teacher.flags must be"),
                           (TeacherForcing(fr, [0] * b), "teacher.flags must be")):
        with pytest.raises(ValueError, match=match):
            m.rollout(x, cp, mk, K, teacher=teacher)
    with pytest.raises(ValueError, match="steps >= 2"):
        m.rollout(x, cp, mk, 1, teacher=TeacherForcing(fr[:0], fl[:0]))
    for teacher in (None, TeacherForcing(fr, fl), TeacherForcing(fr, fl.bool())):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            m.rollout(x, cp, mk, K, teacher=teacher)


def test_teacher_forcing_flags_rejects_bad_arguments():
    ids = torch.zeros(3, dtype=torch.int64)
    for kw, match in ((dict(steps=1), "steps must be"), (dict(steps=2 ** 16 + 1), "steps must be"),
                      (dict(steps=3.0), "steps must be"), (dict(prob=-0.1), r"prob must be a real number in \[0, 1\]"),
                      (dict(prob=1.5), "prob must be"), (dict(prob=float("nan")), "prob must be"),
                      (dict(prob=True), "prob must be"), (dict(seed=-1), "seed must be"), (dict(seed=2 ** 64), "seed"),
                      (dict(step=-1), "step must be"), (dict(step=1.0), "step must be"),
                      (dict(ids=ids.int()), "ids must be"), (dict(ids=ids[:0]), "ids must be"),
                      (dict(ids=ids[None]), "ids must be"), (dict(), "CUDA device")):
        args = dict(ids=ids, steps=3, prob=0.5, seed=1, step=1)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            teacher_forcing_flags(**args)


def test_train_auto_rejects_bad_teacher_arguments_before_the_cpu_refusal(tmp_path):
    out = tmp_path / "out"
    tr, dv = _TimedSplit(12), _Split(3)
    m = _cpu_model()
    for tf, match in ((-0.1, "teacher_forcing must be a real number in"), (1.01, "teacher_forcing must be"),
                      (float("nan"), "teacher_forcing must be"), (float("inf"), "teacher_forcing must be"),
                      (True, "teacher_forcing must be None"), ("0.5", "teacher_forcing must be None"),
                      ([0.5, 0.4], "fewer than num_epochs=3"), ([0.5, 0.4, 2.0], r"teacher_forcing\[2\] must be"),
                      (object(), "teacher_forcing must be None")):
        with pytest.raises(ValueError, match=match):
            train_auto(m, tr, dv, out, num_epochs=3, rollout_steps=3, teacher_forcing=tf)
    for seed in (-1, 2 ** 64, 1.0, True, "3"):
        with pytest.raises(ValueError, match="teacher_seed must be an int"):
            train_auto(m, tr, dv, out, num_epochs=3, rollout_steps=3, teacher_forcing=0.5, teacher_seed=seed)
    for kw, match in ((dict(), "needs rollout_steps > 1"), (dict(rollout_steps=1), "needs rollout_steps > 1"),
                      (dict(rollout_steps=3, rollout_grad_steps=1), "does not combine with pushforward"),
                      (dict(rollout_steps=3, rollout_grad_steps=2, random_unroll=True), "does not combine")):
        with pytest.raises(ValueError, match=match):
            train_auto(m, tr, dv, out, num_epochs=3, teacher_forcing=0.5, **kw)
    # valid set-ups get as far as the CPU model's refusal
    for kw in (dict(teacher_forcing=0.5), dict(teacher_forcing=0), dict(teacher_forcing=np.float32(1.0)),
               dict(teacher_forcing=[1.0, 0.5, 0.0, 7.0][:3], teacher_seed=2 ** 64 - 1),
               dict(teacher_forcing=np.linspace(1, 0, 5), teacher_seed=np.uint64(3), input_noise_std=0.1,
                    noise_every_step=True, max_grad_norm=1.0, ema_decay=0.9), dict(teacher_forcing=None)):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            train_auto(m, tr, dv, out, num_epochs=3, rollout_steps=3, **kw)
    assert not out.exists()   # rejected before anything was written


def test_resume_refuses_a_changed_teacher_setting_by_name(tmp_path):
    m, tr, dv = _cpu_model(), _TimedSplit(12), _Split(3)
    rollout = dict(DEFAULTS, rollout_steps=3, rollout_grad_steps=3, time_step_size=1)
    out = tmp_path / "run"
    out.mkdir()
    resume.write_state(_state(m, resume.run_config(m, tr, dv, **rollout, teacher_forcing=[1.0, 0.5], teacher_seed=5)),
                       out)
    call = dict(rollout_steps=3, resumable=True, num_epochs=2)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):   # the same call gets past the state
        train_auto(m, tr, dv, out, teacher_forcing=(1.0, 0.5), teacher_seed=5, **call)
    for kw, fields in ((dict(teacher_forcing=[1.0, 0.4], teacher_seed=5), ["teacher_forcing"]),
                       (dict(teacher_forcing=[1.0, 0.5], teacher_seed=6), ["teacher_seed"]),
                       (dict(teacher_forcing=0.5, teacher_seed=5), ["teacher_forcing"]),
                       (dict(), ["teacher_forcing", "teacher_seed"])):
        with pytest.raises(ValueError, match="other settings") as e:
            train_auto(m, tr, dv, out, **call, **kw)
        assert [f.split(":")[0] for f in str(e.value).split("Differing: ")[1].split("; ")] == fields, kw
    assert "teacher_forcing: saved [1.0, 0.5], now (absent)" in str(e.value)
    # a run without teacher forcing records neither field, and refuses a teacher-forced relaunch
    plain = tmp_path / "plain"
    plain.mkdir()
    resume.write_state(_state(m, resume.run_config(m, tr, dv, **rollout)), plain)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, dv, plain, **call)
    with pytest.raises(ValueError, match=r"Differing: teacher_forcing: saved \(absent\), now 0.5; teacher_seed: saved "
                                         r"\(absent\), now 0$"):
        train_auto(m, tr, dv, plain, teacher_forcing=0.5, **call)
