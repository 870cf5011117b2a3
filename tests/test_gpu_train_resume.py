"""Resumable `train_auto` runs on the GPU: a run interrupted and resumed with `resumable=True` equals the run that was
never interrupted, bit for bit (parameters, optimizer state, losses, norms, EMA, every checkpoint and JSON file); a
finished run relaunched trains nothing and extended equals a longer straight run; a changed call is refused before
any file changes; the default writes no state; and the time of one state write at cavity size."""
import json
import statistics
import time

import pytest
import torch

from cfdbench_b200 import resume, train_auto
from test_gpu_eval_auto import _AutoSplit, _model
from test_gpu_train_rollout import _ChainSplit

pytestmark = pytest.mark.gpu

# problem, storage, splits, train_auto arguments (generator: True for an explicit one, None for the global RNG)
CONFIGS = {
    "cavity-fp32-single": ("cavity", "float32", lambda: (_AutoSplit(19, "cavity", seed=21), _AutoSplit(4, "cavity", seed=22)),
                           dict(batch_size=8, eval_interval=2, generator=True)),
    "cavity-bf16-rollout-stabilised": (
        "cavity", "bfloat16", lambda: (_ChainSplit((9, 12, 7), "cavity", s=1, seed=31),
                                       _ChainSplit((8, 6), "cavity", s=1, seed=32)),
        dict(batch_size=8, eval_interval=2, rollout_steps=3, rollout_grad_steps=2, input_noise_std=0.05, noise_seed=77,
             noise_every_step=True, max_grad_norm=0.02, ema_decay=0.99, dev_rollout_steps=2, generator=None)),
    "tube-pushforward-noise": ("tube", "float32", lambda: (_ChainSplit((9, 12, 7), "tube", s=1, seed=41),
                                                           _AutoSplit(4, "tube", seed=42)),
                               dict(batch_size=8, eval_interval=3, rollout_steps=3, rollout_grad_steps=1,
                                    input_noise_std=0.05, noise_seed=5, generator=True)),
}


def _call(name, splits, out, epochs, model_seed=8, rng_seed=5, **over):
    """One train_auto call of configuration `name`, on a freshly built model; the visiting order's RNG is seeded with
    rng_seed (a resumed call restores it from the state, whatever it was seeded with)."""
    problem, act_dtype, _, kw = CONFIGS[name]
    kw = dict(kw, **over)
    m = _model(problem, act_dtype, seed=model_seed)   # (draws from the global RNG: seed it afterwards)
    if kw.pop("generator"):
        kw["generator"] = torch.Generator().manual_seed(rng_seed)
    else:
        torch.manual_seed(rng_seed)
    res = train_auto(m, *splits, out, num_epochs=epochs, lr=1e-3, eval_batch_size=3, log_interval=1000,
                     resumable=kw.pop("resumable", True), **kw)
    return m, res


def _equal(a, b, where):
    """Recursive bit equality of loaded state / checkpoint contents."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a.cpu(), b.cpu()), where
    elif isinstance(a, dict):
        assert set(a) == set(b), where
        for k in a:
            _equal(a[k], b[k], f"{where}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, f"{where}[{i}]")
    else:
        assert a == b, (where, a, b)


def _files(out):
    return sorted(str(p.relative_to(out)) for p in out.rglob("*") if p.is_file())


def _assert_same_run(a, b):
    """(model, result, output_dir) of two runs: the same parameters, optimizer state, results and files."""
    (ma, ra, da), (mb, rb, db) = a, b
    for (name, pa), pb in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(pa, pb), name
        sa, sb = ra["optimizer"].state.get(pa), rb["optimizer"].state.get(pb)
        assert (sa is None) == (sb is None), name
        if sa is not None:
            assert set(sa) == set(sb), name
            for k in sa:
                assert torch.equal(sa[k], sb[k]), (name, k)
    assert ra["train_losses"] == rb["train_losses"]
    assert ra.get("grad_norms") == rb.get("grad_norms")
    assert ("ema_model" in ra) == ("ema_model" in rb)
    if "ema_model" in ra:
        for (name, ea), eb in zip(ra["ema_model"].named_parameters(), rb["ema_model"].parameters()):
            assert torch.equal(ea, eb), name
    assert _files(da) == _files(db)
    for f in _files(da):
        if f.endswith(".pt"):   # every ckpt-*/model.pt and the final training state
            _equal(torch.load(da / f, map_location="cpu", weights_only=True),
                   torch.load(db / f, map_location="cpu", weights_only=True), f)
        else:
            ja, jb = json.load(open(da / f)), json.load(open(db / f))
            if f.endswith("scores.json") and "time" in ja:   # the epoch's wall time
                ja.pop("time"), jb.pop("time")
            assert ja == jb, f


@pytest.mark.parametrize("name,epochs,split", [("cavity-fp32-single", 5, 3), ("cavity-bf16-rollout-stabilised", 5, 2),
                                               ("tube-pushforward-noise", 5, 4)])
def test_split_run_equals_straight_run(tmp_path, name, epochs, split):
    splits = CONFIGS[name][2]()
    straight = _call(name, splits, tmp_path / "a", epochs) + (tmp_path / "a",)
    b_dir = tmp_path / "b"
    m1, r1 = _call(name, splits, b_dir, split)
    assert r1["start_epoch"] == 0
    state = torch.load(b_dir / resume.STATE_NAME, map_location="cpu", weights_only=True)
    assert state["epoch"] == split - 1 and state["global_step"] == len(r1["train_losses"])
    torch.rand(7)   # the relaunched process's global RNG is anywhere: the state restores it
    m2, r2 = _call(name, splits, b_dir, epochs, model_seed=99, rng_seed=1234)
    assert r2["start_epoch"] == split
    assert r2["train_losses"][:len(r1["train_losses"])] == r1["train_losses"]
    _assert_same_run(straight, (m2, r2, b_dir))
    n_ckpt = len(list(b_dir.glob("ckpt-*")))
    print(f"{name}: split after epoch {split - 1}, {len(r2['train_losses'])} steps, {n_ckpt} checkpoints: equal")


def test_finished_run_relaunched_and_extended(tmp_path):
    name, over = "cavity-fp32-single", dict(max_grad_norm=0.05, ema_decay=0.9)
    splits = CONFIGS[name][2]()
    out = tmp_path / "run"
    ma, ra = _call(name, splits, out, 5, **over)
    files = {f: ((out / f).read_bytes(), (out / f).stat().st_mtime_ns) for f in _files(out)}
    steps = {k: float(v["step"]) for k, v in ra["optimizer"].state_dict()["state"].items()}
    for epochs in (5, 3):   # no larger than what was trained: no step
        m, r = _call(name, splits, out, epochs, model_seed=99, rng_seed=1, **over)
        assert r["start_epoch"] == 5
        assert {k: float(v["step"]) for k, v in r["optimizer"].state_dict()["state"].items()} == steps
        for (n, a), b in zip(ma.named_parameters(), m.parameters()):
            assert torch.equal(a, b), n
        assert r["train_losses"] == ra["train_losses"] and r["grad_norms"] == ra["grad_norms"]
        for (n, a), b in zip(ra["ema_model"].named_parameters(), r["ema_model"].parameters()):
            assert torch.equal(a, b), n
        assert _files(out) == sorted(files)
        for f, (data, mtime) in files.items():
            assert (out / f).read_bytes() == data, f
            if f not in ("train_losses.json", "grad_norms.json"):   # the only files a finished run rewrites
                assert (out / f).stat().st_mtime_ns == mtime, f
    m, r = _call(name, splits, out, 8, model_seed=98, **over)
    assert r["start_epoch"] == 5
    longer = tmp_path / "longer"
    _assert_same_run(_call(name, splits, longer, 8, **over) + (longer,), (m, r, out))


def test_changed_call_is_refused_before_any_file_changes(tmp_path):
    name = "cavity-fp32-single"
    splits = CONFIGS[name][2]()
    out = tmp_path / "run"
    _call(name, splits, out, 2)
    files = {f: ((out / f).read_bytes(), (out / f).stat().st_mtime_ns) for f in _files(out)}
    m = _model("cavity", seed=3)
    with pytest.raises(ValueError, match=r"Differing: lr: saved 0\.001, now 0\.002"):
        train_auto(m, *splits, out, num_epochs=4, lr=2e-3, batch_size=8, eval_interval=2, eval_batch_size=3,
                   generator=torch.Generator().manual_seed(5), resumable=True)
    assert {f: ((out / f).read_bytes(), (out / f).stat().st_mtime_ns) for f in _files(out)} == files


def test_default_writes_no_state_and_resumable_changes_no_bit(tmp_path):
    name = "cavity-fp32-single"
    splits = CONFIGS[name][2]()
    m0, r0 = _call(name, splits, tmp_path / "default", 3, resumable=False)
    assert not (tmp_path / "default" / resume.STATE_NAME).exists() and r0["start_epoch"] == 0
    assert not list((tmp_path / "default").glob(".*"))
    m1, r1 = _call(name, splits, tmp_path / "resumable", 3)
    assert (tmp_path / "resumable" / resume.STATE_NAME).exists()
    (tmp_path / "resumable" / resume.STATE_NAME).unlink()
    _assert_same_run((m0, r0, tmp_path / "default"), (m1, r1, tmp_path / "resumable"))


def test_state_write_time_at_cavity_size(tmp_path):
    """One state write of the cavity model (4 layers, 32 channels, 12x12 modes: 2,368,354 reals) after training, with
    and without the EMA: its size against weights + moments (+ EMA) in float32, and its time, host copy included."""
    splits = CONFIGS["cavity-fp32-single"][2]()
    reals = sum(p.numel() * (2 if p.is_complex() else 1) for p in _model("cavity").parameters())
    assert reals == 2_368_354
    name = torch.cuda.get_device_name()
    for ema in (None, 0.99):
        out = tmp_path / f"ema-{ema}"
        m, r = _call("cavity-fp32-single", splits, out, 1, ema_decay=ema)
        opt = r["optimizer"]
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.9)
        config = torch.load(out / resume.STATE_NAME, map_location="cpu", weights_only=True)["config"]
        times = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            resume.write_state(resume.build_state(0, 3, m, opt, sched, None, r["train_losses"], None, config), out)
            times.append(time.perf_counter() - t0)
        size = (out / resume.STATE_NAME).stat().st_size
        want = 4 * reals * (3 + (ema is not None))
        assert want <= size < want + 1_000_000, (size, want)
        print(f"state write at cavity size, ema={ema}: {size / 1e6:.1f} MB, median {statistics.median(times) * 1e3:.1f} ms "
              f"(min {min(times) * 1e3:.1f}, max {max(times) * 1e3:.1f}) over 5 writes on {name}")
