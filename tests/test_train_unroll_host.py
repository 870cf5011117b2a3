"""Random pushforward unroll lengths (`train_auto(random_unroll=True)`) without a GPU: `unroll_lengths` -- its range,
its independence of how the steps are split into calls, its seed, its uniformity -- the argument checks, and the
resume config record of the two new arguments."""
import numpy as np
import pytest
import torch

import cfdbench_b200
from cfdbench_b200 import _lib, resume, train_auto, unroll_lengths
from test_train_auto_host import _cpu_model, _Split
from test_train_resume_host import DEFAULTS, _state
from test_train_rollout_host import _TimedSplit


# ------------------------------------------------------------------------------------------------ unroll_lengths
@pytest.mark.parametrize("max_prefix", [1, 3, 7])
def test_values_lie_in_range_and_follow_the_definition(max_prefix):
    u = unroll_lengths(5, 1, 500, max_prefix)
    assert u.dtype == np.int64 and u.shape == (500,)
    assert u.min() == 0 and u.max() == max_prefix
    for t in (1, 2, 250, 500):
        assert u[t - 1] == np.random.default_rng((5, t)).integers(0, max_prefix + 1)
    assert unroll_lengths(5, 1, 0, max_prefix).shape == (0,)


def test_one_call_equals_any_split_of_it():
    whole = unroll_lengths(11, 7, 300, 3)
    rng = np.random.default_rng(0)
    for _ in range(10):
        cuts = np.sort(rng.choice(np.arange(1, 300), size=rng.integers(1, 6), replace=False))
        parts, start = [], 0
        for end in list(cuts) + [300]:
            parts.append(unroll_lengths(11, 7 + start, end - start, 3))
            start = end
        assert np.array_equal(np.concatenate(parts), whole), cuts
    assert np.array_equal(np.concatenate([unroll_lengths(11, t, 1, 3) for t in range(7, 307)]), whole)


def test_different_seeds_give_different_sequences():
    seqs = [unroll_lengths(s, 1, 64, 3) for s in (0, 1, 2, 2 ** 40)]
    for i in range(len(seqs)):
        for j in range(i + 1, len(seqs)):
            assert not np.array_equal(seqs[i], seqs[j]), (i, j)
    assert np.array_equal(unroll_lengths(np.uint64(1), 1, 64, 3), seqs[1])


@pytest.mark.parametrize("max_prefix", [1, 3, 7])
def test_every_value_is_uniform_within_three_sigma(max_prefix):
    n, k = 20_000, max_prefix + 1
    counts = np.bincount(unroll_lengths(3, 1, n, max_prefix), minlength=k)
    assert counts.size == k
    p = 1.0 / k
    sigma = np.sqrt(n * p * (1 - p))
    assert np.all(np.abs(counts - n * p) <= 3 * sigma), (counts, n * p, sigma)


# ------------------------------------------------------------------------------------------------ argument checks
def test_train_auto_rejects_bad_unroll_arguments_before_the_cpu_refusal(tmp_path):
    out = tmp_path / "out"
    tr, dv = _TimedSplit(12), _Split(3)
    m = _cpu_model()
    for bad in (1, 0, "yes", None, np.bool_(True)):
        with pytest.raises(ValueError, match="random_unroll must be a bool"):
            train_auto(m, tr, dv, out, rollout_steps=3, rollout_grad_steps=1, random_unroll=bad)
    for kw in (dict(), dict(rollout_steps=1), dict(rollout_steps=1, rollout_grad_steps=1), dict(rollout_steps=3),
               dict(rollout_steps=3, rollout_grad_steps=3)):
        with pytest.raises(ValueError, match="random_unroll .*rollout_grad_steps < rollout_steps"):
            train_auto(m, tr, dv, out, random_unroll=True, **kw)
    for seed in (-1, 1.0, True, "3", None, np.float64(2)):
        with pytest.raises(ValueError, match="unroll_seed must be a non-negative int"):
            train_auto(m, tr, dv, out, rollout_steps=3, rollout_grad_steps=1, random_unroll=True, unroll_seed=seed)
    # valid set-ups get as far as the CPU model's refusal
    for kw in (dict(rollout_steps=2, rollout_grad_steps=1, random_unroll=True),
               dict(rollout_steps=3, rollout_grad_steps=2, random_unroll=True, unroll_seed=2 ** 70),
               dict(rollout_steps=3, rollout_grad_steps=1, random_unroll=True, unroll_seed=np.uint64(7),
                    input_noise_std=0.1, noise_every_step=True, max_grad_norm=1.0, ema_decay=0.9),
               dict(random_unroll=False, unroll_seed=4), dict(rollout_steps=3, random_unroll=False)):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            train_auto(m, tr, dv, out, **kw)
    assert not out.exists()   # rejected before anything was written
    assert "unroll_lengths" in cfdbench_b200.__all__


# ------------------------------------------------------------------------------------------------ resume record
def test_resume_refuses_a_changed_unroll_setting_by_name(tmp_path):
    m, tr, dv = _cpu_model(), _TimedSplit(12), _Split(3)
    rollout = dict(DEFAULTS, rollout_steps=3, rollout_grad_steps=1, time_step_size=1)
    out = tmp_path / "run"
    out.mkdir()
    resume.write_state(_state(m, resume.run_config(m, tr, dv, **rollout, random_unroll=True, unroll_seed=5)), out)
    call = dict(rollout_steps=3, rollout_grad_steps=1, resumable=True)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):   # the same call gets past the state
        train_auto(m, tr, dv, out, random_unroll=True, unroll_seed=5, **call)
    # a fixed-prefix call records neither field (its record is the one runs without the option always wrote)
    for kw, fields in ((dict(random_unroll=True, unroll_seed=6), ["unroll_seed"]),
                       (dict(random_unroll=False, unroll_seed=5), ["random_unroll", "unroll_seed"]),
                       (dict(), ["random_unroll", "unroll_seed"])):
        with pytest.raises(ValueError, match="other settings") as e:
            train_auto(m, tr, dv, out, **call, **kw)
        assert [f.split(":")[0] for f in str(e.value).split("Differing: ")[1].split("; ")] == fields, kw
    assert "random_unroll: saved True, now (absent)" in str(e.value)
    # and a fixed-prefix run's state refuses a random-unroll relaunch
    fixed = tmp_path / "fixed"
    fixed.mkdir()
    resume.write_state(_state(m, resume.run_config(m, tr, dv, **rollout)), fixed)
    with pytest.raises(_lib.FnoNativeError, match="CPU"):
        train_auto(m, tr, dv, fixed, **call)
    with pytest.raises(ValueError, match=r"Differing: random_unroll: saved \(absent\), now True; unroll_seed: saved "
                                         r"\(absent\), now 0$"):
        train_auto(m, tr, dv, fixed, random_unroll=True, **call)
    cfg = resume.run_config(m, tr, dv, **rollout, random_unroll=True, unroll_seed=5)
    for k, v in (("random_unroll", False), ("unroll_seed", 9)):
        with pytest.raises(ValueError, match=rf"Differing: {k}: saved "):
            resume.check_config(cfg, dict(cfg, **{k: v}), tmp_path)
    assert set(torch.load(out / resume.STATE_NAME, weights_only=True)["config"]) - set(resume.run_config(
        m, tr, dv, **rollout)) == {"random_unroll", "unroll_seed"}
