"""Resumable `train_auto` runs (`train_auto(..., resumable=True)`, cfdbench_b200.resume) without a GPU: every config
field compared on resume, the start-up cases, a state that loads with weights_only=True, the atomic write, and the
visiting order continued from a state taken at an epoch boundary."""
import os
import warnings

import numpy as np
import pytest
import torch

from cfdbench_b200 import FusedAdam, _lib, resume, train_auto
from cfdbench_b200.train import dev_eval_draw, index_stream
from test_train_auto_host import _cpu_model, _Split

# what train_auto resolves for its defaults on a single-step run: the config record of such a call
DEFAULTS = dict(lr=1e-3, lr_step_size=1, lr_gamma=0.9, batch_size=2, eval_batch_size=2, eval_interval=2, rollout_steps=1,
                time_step_size=None, rollout_grad_steps=1, input_noise_std=0.0, noise_seed=0, noise_every_step=False,
                dev_rollout_steps=None, dev_time_step_size=None, max_grad_norm=None, ema_decay=None, generator=False)
MODEL_FIELDS = ("in_chan", "out_chan", "n_case_params", "num_layers", "hidden_dim", "modes1", "modes2", "act_dtype",
                "fused_block", "generic_grid_at_64", "requires_grad")
SPLIT_FIELDS = ("n", "height", "width", "n_case_params", "frame_dtype", "case_ids_sha256")


def _splits():
    tr, dv = _Split(6), _Split(3)
    tr.case_ids = np.asarray([0, 0, 0, 1, 1, 1])
    return tr, dv


def _state(model, config, generator=None, ema=True, steps=3):
    """A complete state of `model` after `steps` fake Adam steps, built by the helper train_auto uses."""
    opt = FusedAdam(model.parameters(), lr=config["lr"], ema_decay=0.9 if ema else None)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.9)
    g = torch.Generator().manual_seed(11)
    for p in model.parameters():
        st = opt.init_state(p)
        st["step"] += steps
        for k in ("exp_avg", "exp_avg_sq") + (("ema",) if ema else ()):
            st[k].copy_(torch.randn(p.shape, dtype=p.dtype, generator=g))
    with warnings.catch_warnings():   # no optimizer.step() ran: the steps are fake
        warnings.simplefilter("ignore")
        for _ in range(steps):
            sched.step()
    return resume.build_state(2, steps, model, opt, sched, generator, [0.5, 0.25, 0.125], [1.5, 2.5, 3.5], config)


# ------------------------------------------------------------------------------------------------ the config record
def test_config_holds_every_field():
    m, (tr, dv) = _cpu_model(), _splits()
    cfg = resume.run_config(m, tr, dv, **DEFAULTS)
    want = {f"model.{k}" for k in MODEL_FIELDS} | set(DEFAULTS) | \
        {f"{s}.{k}" for s in ("train_data", "dev_data") for k in SPLIT_FIELDS}
    assert set(cfg) == want
    assert cfg["model.requires_grad"] == [True] * len(list(m.parameters()))
    assert cfg["train_data.n"] == 6 and cfg["train_data.frame_dtype"] == "float32"


def _changed(v):
    if isinstance(v, bool):
        return not v
    if v is None:
        return 3
    if isinstance(v, (int, float)):
        return v * 2 + 1
    if isinstance(v, str):
        return v + "x"
    if isinstance(v, list):
        return v[:-1] + [not v[-1]]
    raise AssertionError(v)


def test_each_field_changed_alone_is_refused_by_name(tmp_path):
    m, (tr, dv) = _cpu_model(), _splits()
    cfg = resume.run_config(m, tr, dv, **DEFAULTS)
    resume.check_config(cfg, dict(cfg), tmp_path)
    for k in cfg:
        other = dict(cfg)
        other[k] = _changed(cfg[k])
        with pytest.raises(ValueError, match=rf"Differing: {k}: saved "):
            resume.check_config(cfg, other, tmp_path)
    other = dict(cfg, lr=5.0, batch_size=7)
    del other["ema_decay"]
    with pytest.raises(ValueError, match=r"batch_size: saved 2, now 7; ema_decay: saved None, now \(absent\); lr: saved"):
        resume.check_config(cfg, other, tmp_path)


def test_split_fingerprint_sees_each_field():
    base = _Split(6)
    fp = resume.split_fingerprint(base)
    permuted = _Split(6)
    permuted.case_ids = np.asarray([0, 0, 0, 0, 0, 1])
    for data, field in ((_Split(6, gh=66), "height"), (_Split(6, gw=65), "width"), (_Split(6, p=4), "n_case_params"),
                        (permuted, "case_ids_sha256")):
        got = resume.split_fingerprint(data)
        assert [k for k in fp if fp[k] != got[k]] == [field], field
    got = resume.split_fingerprint(_Split(7))
    assert [k for k in fp if fp[k] != got[k]] == ["n", "case_ids_sha256"]
    # a DeviceFrames in bf16 storage differs in frame_dtype only (stands in without a device: same attributes)
    frames = resume.DeviceFrames.__new__(resume.DeviceFrames)
    frames.n, frames.height, frames.width, frames.n_case_params = 6, 64, 64, 5
    frames.frame_dtype, frames._case_ids_host = torch.bfloat16, base.case_ids
    got = resume.split_fingerprint(frames)
    assert [k for k in fp if fp[k] != got[k]] == ["frame_dtype"] and got["frame_dtype"] == "bfloat16"


# train_auto arguments changed alone -> the config fields they must change
CALL_CHANGES = [
    (dict(lr=2e-3), ["lr"]), (dict(lr_step_size=2), ["lr_step_size"]), (dict(lr_gamma=0.5), ["lr_gamma"]),
    (dict(batch_size=3), ["batch_size"]), (dict(eval_batch_size=3), ["eval_batch_size"]),
    (dict(eval_interval=3), ["eval_interval"]), (dict(input_noise_std=0.1), ["input_noise_std"]),
    (dict(noise_seed=5), ["noise_seed"]), (dict(noise_every_step=True), ["noise_every_step"]),
    (dict(max_grad_norm=1.0), ["max_grad_norm"]), (dict(ema_decay=0.99), ["ema_decay"]),
    (dict(generator=torch.Generator()), ["generator"]),
    (dict(rollout_steps=2, time_step_size=1), ["rollout_grad_steps", "rollout_steps", "time_step_size"]),
    (dict(rollout_steps=3, rollout_grad_steps=1, time_step_size=1), ["rollout_steps", "time_step_size"]),
    (dict(dev_rollout_steps=2, time_step_size=1), ["dev_rollout_steps", "dev_time_step_size"]),
]


def test_train_auto_refuses_a_changed_call_before_any_device_work(tmp_path):
    m, (tr, dv) = _cpu_model(), _splits()
    out = tmp_path / "run"
    out.mkdir()
    resume.write_state(_state(m, resume.run_config(m, tr, dv, **DEFAULTS)), out)
    before = (out / resume.STATE_NAME).read_bytes()
    # num_epochs and log_interval are free: the call gets past the state to the CPU-model refusal
    for kw in (dict(), dict(num_epochs=1000), dict(log_interval=1)):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            train_auto(m, tr, dv, out, resumable=True, **kw)
    for kw, fields in CALL_CHANGES:
        with pytest.raises(ValueError, match="other settings") as e:
            train_auto(m, tr, dv, out, resumable=True, **kw)
        named = [f.split(":")[0] for f in str(e.value).split("Differing: ")[1].split("; ")]
        assert named == fields, (kw, named)
    frozen = _cpu_model()
    next(frozen.parameters()).requires_grad_(False)
    bf16 = _cpu_model(act_dtype="bfloat16")
    bf16.fused_block = False
    shorter, reordered = _Split(5), _splits()[0]
    reordered.case_ids = reordered.case_ids[::-1].copy()
    for args, fields in (((frozen, tr, dv), ["model.requires_grad"]),
                         ((bf16, tr, dv), ["model.act_dtype", "model.fused_block"]),
                         ((m, shorter, dv), ["train_data.case_ids_sha256", "train_data.n"]),
                         ((m, reordered, dv), ["train_data.case_ids_sha256"]),
                         ((m, tr, _Split(3, p=5, gh=66, gw=65)), ["dev_data.height", "dev_data.width"])):
        with pytest.raises(ValueError, match="other settings") as e:
            train_auto(*args, out, resumable=True)
        assert [f.split(":")[0] for f in str(e.value).split("Differing: ")[1].split("; ")] == fields
    assert os.listdir(out) == [resume.STATE_NAME] and (out / resume.STATE_NAME).read_bytes() == before


# ------------------------------------------------------------------------------------------------ start-up cases
def test_start_up_cases(tmp_path):
    m, (tr, dv) = _cpu_model(), _splits()
    cfg = resume.run_config(m, tr, dv, **DEFAULTS)
    fresh = tmp_path / "fresh"
    assert resume.find_state(fresh, cfg) is None
    with pytest.raises(_lib.FnoNativeError, match="CPU"):   # no state, no checkpoint: a fresh start
        train_auto(m, tr, dv, fresh, resumable=True)
    fresh.mkdir()
    assert resume.find_state(fresh, cfg) is None
    old = tmp_path / "old"
    (old / "ckpt-3").mkdir(parents=True)
    (old / "ckpt-3" / "model.pt").write_bytes(b"weights")
    with pytest.raises(ValueError, match=r"holds checkpoints \(ckpt-3\) but no training_state.pt"):
        train_auto(m, tr, dv, old, resumable=True)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):   # resumable=False is not concerned with the directory
        train_auto(m, tr, dv, old)
    with pytest.raises(ValueError, match="resumable must be a bool"):
        train_auto(m, tr, dv, fresh, resumable=1)
    (old / resume.STATE_NAME).write_bytes(b"not a state")
    with pytest.raises(ValueError, match="not a readable training state"):
        resume.find_state(old, cfg)
    st = _state(m, cfg)
    st["version"] = resume.STATE_VERSION + 1
    torch.save(st, old / resume.STATE_NAME)
    with pytest.raises(ValueError, match="format version"):
        resume.find_state(old, cfg)
    resume.write_state(_state(m, cfg), old)
    got = resume.find_state(old, cfg)
    assert got["epoch"] == 2 and got["global_step"] == 3 and got["config"] == cfg


# ------------------------------------------------------------------------------------------------ the state file
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("explicit", [False, True])
def test_state_loads_with_weights_only(tmp_path, ema, explicit):
    m, (tr, dv) = _cpu_model(), _splits()
    cfg = resume.run_config(m, tr, dv, **dict(DEFAULTS, generator=explicit, ema_decay=0.9 if ema else None))
    gen = torch.Generator().manual_seed(4) if explicit else None
    st = _state(m, cfg, generator=gen, ema=ema)
    path = resume.write_state(st, tmp_path)
    got = torch.load(path, map_location="cpu", weights_only=True)
    assert set(got) == {"version", "epoch", "global_step", "model", "optimizer", "scheduler", "rng", "rng_state",
                        "train_losses", "grad_norms", "config"}
    assert got["rng"] == ("generator" if explicit else "global")
    assert torch.equal(got["rng_state"], gen.get_state() if explicit else torch.get_rng_state())
    assert got["train_losses"] == [0.5, 0.25, 0.125] and got["grad_norms"] == [1.5, 2.5, 3.5]
    for k, v in m.state_dict().items():
        assert torch.equal(got["model"][k], v) and got["model"][k].dtype == v.dtype, k
    assert got["scheduler"]["last_epoch"] == 3 and got["scheduler"]["_last_lr"] == st["scheduler"]["_last_lr"]
    # the optimizer state loads back into a fresh FusedAdam (complex state stays complex) and into torch.optim.Adam
    fresh = _cpu_model()
    opt = FusedAdam(fresh.parameters(), lr=1.0, ema_decay=0.9 if ema else None)
    opt.load_state_dict(got["optimizer"])
    for i, (p, q) in enumerate(zip(m.parameters(), fresh.parameters())):
        a, b = got["optimizer"]["state"][i], opt.state[q]
        assert b["exp_avg"].dtype == p.dtype and torch.equal(a["exp_avg_sq"], b["exp_avg_sq"])
        assert float(b["step"]) == 3 and ("ema" in b) == ema
    assert opt.param_groups[0]["lr"] == st["optimizer"]["param_groups"][0]["lr"]
    # the host copy is a copy: changing the live state afterwards leaves the built state alone
    live = FusedAdam(m.parameters())
    sched = torch.optim.lr_scheduler.StepLR(live, step_size=1)
    name0, p0 = next(iter(m.named_parameters()))
    live.init_state(p0)
    built = resume.build_state(0, 1, m, live, sched, gen, [], None, cfg)
    with torch.no_grad():
        p0.add_(1.0)
    live.state[p0]["step"] += 1
    assert not torch.equal(built["model"][name0], p0)
    assert float(built["optimizer"]["state"][0]["step"]) == 0 and "grad_norms" not in built


def test_write_is_atomic(tmp_path, monkeypatch):
    m, (tr, dv) = _cpu_model(), _splits()
    cfg = resume.run_config(m, tr, dv, **DEFAULTS)
    path = resume.write_state(_state(m, cfg, steps=3), tmp_path)
    before = path.read_bytes()
    real_save = torch.save

    def killed_save(obj, f, *a, **kw):   # writes a prefix of the new state, then fails
        real_save(obj, f, *a, **kw)
        f.seek(len(before) // 3)
        f.truncate()
        raise OSError("no space left on device")
    monkeypatch.setattr(torch, "save", killed_save)
    with pytest.raises(OSError, match="no space"):
        resume.write_state(_state(m, cfg, steps=5), tmp_path)
    monkeypatch.undo()
    assert os.listdir(tmp_path) == [resume.STATE_NAME]   # no partial file, under any name
    assert path.read_bytes() == before
    assert resume.find_state(tmp_path, cfg)["global_step"] == 3
    resume.write_state(_state(m, cfg, steps=5), tmp_path)   # the next write replaces it
    assert os.listdir(tmp_path) == [resume.STATE_NAME] and resume.find_state(tmp_path, cfg)["global_step"] == 5


# ------------------------------------------------------------------------------------------------ the visiting order
@pytest.mark.parametrize("n,batch_size", [(23, 4), (8, 8), (5, 2)])
@pytest.mark.parametrize("split", [1, 4, 5, 6])
@pytest.mark.parametrize("explicit", [False, True])
def test_index_stream_resumed_from_a_state_equals_the_uninterrupted_stream(tmp_path, n, batch_size, split, explicit):
    """With eval_interval 3 epochs 2, 5 and 8 draw an evaluation seed.  A run split after epoch split - 1 (an
    evaluation epoch only for split = 6) continues from the RNG state taken there, through a written and reloaded
    state file, into the stream of the run that was never split."""
    epochs, eval_interval, seed = 9, 3, 123
    m, (tr, dv) = _cpu_model(), _splits()
    cfg = resume.run_config(m, tr, dv, **dict(DEFAULTS, generator=explicit))

    def rng():
        if explicit:
            return torch.Generator().manual_seed(seed)
        torch.manual_seed(seed)
        return None
    g = rng()
    straight = index_stream(n, batch_size, epochs, eval_interval, g)
    after_straight = torch.rand(4, generator=g)
    g = rng()
    first = index_stream(n, batch_size, split, eval_interval, g)
    resume.write_state(_state(m, cfg, generator=g), tmp_path)
    torch.rand(17)   # a relaunched process's RNG is anywhere
    other = torch.Generator().manual_seed(999) if explicit else None
    if other is not None:
        dev_eval_draw(other)
    state = resume.find_state(tmp_path, cfg)
    resume.restore_rng(state, other)
    rest = index_stream(n, batch_size, epochs, eval_interval, other, start_epoch=split)
    assert len(first) == split and len(rest) == epochs - split
    for a, b in zip(first + rest, straight):
        assert np.array_equal(a, b)
    assert torch.equal(torch.rand(4, generator=other), after_straight)
