"""Random pushforward unroll lengths on the GPU: `train_auto(random_unroll=True)` bit for bit against the eager loop a
user writes with `unroll_lengths` + `DeviceFrames.rollout_batch` + `generate_many` + `Fno2d.rollout` (with input noise,
noise on every rollout step, clipping and the EMA), the visiting order of the fixed-prefix call, a resumed run against
the straight run, one synchronisation per epoch and the memory of the fixed-prefix call, and a record of the rollout
error it gives."""
import numpy as np
import pytest
import torch

from cfdbench_b200 import DeviceFrames, FusedAdam, RolloutNoise, add_input_noise, resume, rollout_windows, train_auto, \
    unroll_lengths
from test_gpu_eval_auto import _AutoSplit, _model
from test_gpu_train_pushforward import _Dynamics
from test_gpu_train_resume import _assert_same_run
from test_gpu_train_rollout import _ChainSplit, _count_syncs

pytestmark = pytest.mark.gpu


def _eager_loop(model, frames, windows, K, G, sigma, noise_seed, every, unroll_seed, num_epochs, lr, lr_gamma,
                batch_size, eval_interval, generator, **opts):
    """The loop of train_auto's docstring (INTEGRATION §3) with u = unroll_lengths(unroll_seed, t, 1, K - G)[0]
    prefix steps, FusedAdam(**opts), a real StepLR and the evaluation loader's RNG draw."""
    from cfdbench_b200.data import index_batches
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr, **opts)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=lr_gamma)
    losses, norms, t = [], [], 0
    for ep in range(num_epochs):
        for ib in index_batches(len(windows), batch_size, True, generator):
            t += 1
            u = int(unroll_lengths(unroll_seed, t, 1, K - G)[0])
            b = frames.rollout_batch(windows[ib], K, noise_std=sigma, noise_seed=noise_seed, noise_step=t)
            ids = torch.as_tensor(windows[ib], device="cuda")
            x, rn = b["inputs"], None
            if every:
                for k in range(u):
                    if k > 0:
                        x = add_input_noise(x, b["mask"], ids, sigma, noise_seed, t, stream=k)
                    with torch.no_grad():
                        x = model.generate_many(x, b["case_params"], b["mask"], 1)[0]
                rn = RolloutNoise(sigma, noise_seed, t, ids, u)
            elif u:
                with torch.no_grad():
                    x = model.generate_many(x, b["case_params"], b["mask"], u)[-1]
            seq = model.rollout(x, b["case_params"], b["mask"], G, noise=rn)
            loss = sum(model.loss_fn(preds=seq[g], labels=b["labels"][u + g])["nmse"] for g in range(G)) / G
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss.item())
            if opt.max_grad_norm is not None:
                norms.append(float(opt.last_grad_norm))
        sched.step()
        if (ep + 1) % eval_interval == 0:
            dev_eval_draw(generator)
    return losses, norms, opt


# problem, act_dtype, case lengths, batch_size: every (K, G) below leaves a ragged last batch
CONFIGS = {"cavity-f32": ("cavity", "float32", (9, 15, 7), 8), "cavity-bf16": ("cavity", "bfloat16", (12, 10), 4),
           "tube": ("tube", "float32", (9, 8, 10), 8)}


def _covering_seed(steps, max_prefix):
    """The first unroll seed under which `steps` steps draw every prefix length 0 .. max_prefix."""
    return next(s for s in range(1000) if np.unique(unroll_lengths(s, 1, steps, max_prefix)).size == max_prefix + 1)


def _graph_vs_eager(tmp_path, config, K, G, sigma=0.0, every=False, epochs=4, **opts):
    problem, act_dtype, lengths, batch_size = CONFIGS[config]
    eval_interval, noise_seed, lr_gamma = 2, 2 ** 63 + 9, 0.9
    ds, dev = _ChainSplit(lengths, problem, s=1, seed=31), _AutoSplit(4, problem, seed=32)
    windows = rollout_windows(ds.case_ids, K, 1)
    assert len(windows) % batch_size != 0, "the split must leave a ragged last batch"
    steps = epochs * -(-len(windows) // batch_size)
    seed = _covering_seed(steps, K - G)
    assert set(unroll_lengths(seed, 1, steps, K - G)) == set(range(K - G + 1))
    ref_m, m = _model(problem, act_dtype, seed=8), _model(problem, act_dtype, seed=8)
    ref_losses, ref_norms, ref_opt = _eager_loop(ref_m, DeviceFrames(ds, device="cuda"), windows, K, G, sigma,
                                                 noise_seed, every, seed, epochs, 1e-3, lr_gamma, batch_size,
                                                 eval_interval, torch.Generator().manual_seed(5), **opts)
    out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, lr_gamma=lr_gamma, batch_size=batch_size,
                     eval_batch_size=3, eval_interval=eval_interval, rollout_steps=K, rollout_grad_steps=G,
                     input_noise_std=sigma, noise_seed=noise_seed, noise_every_step=every, random_unroll=True,
                     unroll_seed=seed, generator=torch.Generator().manual_seed(5), **opts)
    losses, opt = out["train_losses"], out["optimizer"]
    assert len(losses) == len(ref_losses) == steps
    print(f"{config} K={K} G={G} sigma={sigma} every={every} {opts}: unroll seed {seed}, max |loss diff| "
          f"{max(abs(a - b) for a, b in zip(losses, ref_losses)):.3e}")
    assert losses == ref_losses
    if "max_grad_norm" in opts:
        assert out["grad_norms"] == ref_norms
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        sa, sb = opt.state[a], ref_opt.state[b]
        for k in ("exp_avg", "exp_avg_sq", "step") + (("ema",) if "ema_decay" in opts else ()):
            assert torch.equal(sa[k], sb[k]), (name, k)
        assert float(sa["step"]) == steps
    assert opt.param_groups[0]["lr"] == ref_opt.param_groups[0]["lr"]


@pytest.mark.parametrize("K,G", [(2, 1), (4, 1), (4, 2)])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_random_unroll_is_bit_identical_to_the_eager_loop(tmp_path, config, K, G):
    _graph_vs_eager(tmp_path, config, K, G)


@pytest.mark.parametrize("K,G,every", [(4, 1, False), (4, 1, True), (4, 2, True)])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_random_unroll_with_noise_is_bit_identical_to_the_eager_loop(tmp_path, config, K, G, every):
    _graph_vs_eager(tmp_path, config, K, G, sigma=0.05, every=every)


def test_random_unroll_with_clipping_and_ema_is_bit_identical_to_the_eager_loop(tmp_path):
    _graph_vs_eager(tmp_path, "cavity-f32", 4, 1, sigma=0.05, every=True, max_grad_norm=0.02, ema_decay=0.99)


# ------------------------------------------------------------------------------------------------ visiting order
def test_visiting_order_is_the_fixed_prefix_calls(tmp_path):
    ds, dev = _ChainSplit((9, 15, 7), "cavity", s=1, seed=1), _AutoSplit(4, "cavity", seed=2)
    gens, outs, models = [], [], []
    for i, kw in enumerate((dict(), dict(random_unroll=False, unroll_seed=7), dict(random_unroll=True, unroll_seed=7))):
        gen = torch.Generator().manual_seed(4)
        m = _model("cavity", seed=3)
        outs.append(train_auto(m, ds, dev, tmp_path / str(i), num_epochs=5, batch_size=8, eval_interval=2,
                               rollout_steps=4, rollout_grad_steps=1, generator=gen, **kw))
        gens.append(gen.get_state())
        models.append(m)
    assert torch.equal(gens[0], gens[1]) and torch.equal(gens[0], gens[2])
    # random_unroll=False is the fixed-prefix call whatever the seed; random_unroll=True trains something else
    assert outs[0]["train_losses"] == outs[1]["train_losses"] != outs[2]["train_losses"]
    for a, b in zip(models[0].parameters(), models[1].parameters()):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ resume
def test_resumed_random_unroll_run_equals_the_straight_run(tmp_path):
    ds, dev = _ChainSplit((9, 12, 7), "cavity", s=1, seed=31), _ChainSplit((8, 6), "cavity", s=1, seed=32)

    def call(out, epochs, model_seed, rng_seed):
        m = _model("cavity", "bfloat16", seed=model_seed)
        torch.manual_seed(rng_seed)   # the global RNG: a resumed call restores it from the state
        return m, train_auto(m, ds, dev, out, num_epochs=epochs, lr=1e-3, batch_size=8, eval_batch_size=3,
                             eval_interval=2, log_interval=1000, rollout_steps=4, rollout_grad_steps=2,
                             input_noise_std=0.05, noise_seed=77, noise_every_step=True, max_grad_norm=0.02,
                             ema_decay=0.99, dev_rollout_steps=2, random_unroll=True, unroll_seed=3, resumable=True)
    straight = call(tmp_path / "a", 5, 8, 5) + (tmp_path / "a",)
    m1, r1 = call(tmp_path / "b", 2, 8, 5)   # interrupted after the evaluation of epoch 1
    state = torch.load(tmp_path / "b" / resume.STATE_NAME, map_location="cpu", weights_only=True)
    assert state["epoch"] == 1 and state["config"]["random_unroll"] is True and state["config"]["unroll_seed"] == 3
    torch.rand(7)
    m2, r2 = call(tmp_path / "b", 5, 99, 1234)
    assert r2["start_epoch"] == 2
    _assert_same_run(straight, (m2, r2, tmp_path / "b"))


# ------------------------------------------------------------------------------------------------ syncs, memory
def test_random_unroll_syncs_once_per_epoch_and_keeps_the_fixed_prefix_memory(tmp_path):
    m = _model("cavity", act_dtype="bfloat16", seed=6)
    dev = DeviceFrames(_AutoSplit(4, "cavity", seed=1), device="cuda")
    tr = DeviceFrames(_ChainSplit((20, 24, 22), "cavity", seed=2), device="cuda")

    def run(epochs, random_unroll):
        return train_auto(m, tr, dev, tmp_path, num_epochs=epochs, batch_size=8, eval_interval=1000, rollout_steps=4,
                          rollout_grad_steps=1, input_noise_std=0.01, noise_seed=1, noise_every_step=True,
                          random_unroll=random_unroll)
    run(1, True)
    counts = {e: len(_count_syncs(lambda: run(e, True))) for e in (1, 3)}
    assert counts == {1: 2, 3: 4}   # the chain check, then one per epoch

    def rise(random_unroll):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(2, random_unroll)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    fixed, rand = rise(False), rise(True)
    print(f"peak rise: fixed prefix {fixed} B, random prefix {rand} B")
    assert rand <= fixed + 2 ** 20


# ------------------------------------------------------------------------------------------------ accuracy record
def test_record_rollout_error_of_random_unroll(tmp_path):
    """One seeded run per mode in the protocol of test_record_rollout_error_of_each_training_mode: K = 4, G = 1, fixed
    against random prefix length, the 1-step and 20-step infer_multistep NMSE.  A record, not a ranking."""
    from cfdbench_b200 import infer_multistep
    tr, test = _Dynamics(6, 24, seed=1), _Dynamics(3, 22, seed=2)
    modes = {"K=4 G=1": dict(rollout_steps=4, rollout_grad_steps=1),
             "K=4 G=1 random": dict(rollout_steps=4, rollout_grad_steps=1, random_unroll=True)}
    for i, (name, kw) in enumerate(modes.items()):
        m = _model("cavity", seed=5)
        train_auto(m, tr, test, tmp_path / str(i), num_epochs=8, batch_size=8, eval_interval=1000,
                   generator=torch.Generator().manual_seed(0), **kw)
        cps = [torch.tensor([0.1 * j for j in range(5)]) for _ in test.all_features]
        nmse = [r["nmse"] for r in infer_multistep(m, test.all_features, cps, infer_steps=20)]
        print(f"ACCURACY {name}: nmse step 1 {nmse[0]:.4g}, step 20 {nmse[-1]:.4g}, mean {np.mean(nmse):.4g}")
        assert np.all(np.isfinite(nmse))
