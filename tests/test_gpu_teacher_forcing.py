"""Teacher forcing of a rollout on the GPU: the flag kernel against its host restatement, `Fno2d.rollout(teacher=...)`
against the rollout without a teacher (all flags 0), one-step rollouts from the true frames (all flags 1) and the float64
oracle (mixed flags), NaN containment, `train_auto(teacher_forcing=...)` bit for bit against its eager loop, its
synchronisations, memory and resume, and a record of the rollout error it gives."""
import numpy as np
import pytest
import torch

from cfdbench_b200 import DeviceFrames, FusedAdam, RolloutNoise, TeacherForcing, resume, rollout_windows, \
    teacher_forcing_flags, train_auto
from test_gpu_eval_auto import _AutoSplit, _model as _auto_model
from test_gpu_rollout_train import CHAINED_BAR, _case, _max_rel, _model, _rel, _report, backward_bar
from test_gpu_train_pushforward import _Dynamics
from test_gpu_train_resume import _assert_same_run
from test_gpu_train_rollout import _ChainSplit, _count_syncs
from test_gpu_train_unroll import CONFIGS
from test_teacher_forcing_host import teacher_flags_reference, teacher_rollout_vjp

pytestmark = pytest.mark.gpu

WHERE = {"cavity-f32": ("cavity", "float32"), "cavity-bf16": ("cavity", "bfloat16"), "tube": ("tube", "float32")}


# ------------------------------------------------------------------------------------------------ the flag kernel
def test_flag_kernel_matches_the_host_restatement():
    ids = torch.arange(0, 3000 * 7919, 7919, dtype=torch.int64, device="cuda")
    for seed, step, steps, p in ((0, 1, 2, 0.5), (2 ** 63 + 9, 2 ** 40 + 3, 5, 0.3), (7, 12, 9, 0.0), (7, 12, 9, 1.0),
                                 (1, 2, 4, 0.999)):
        got = teacher_forcing_flags(ids, steps, p, seed, step).cpu().numpy()
        np.testing.assert_array_equal(got, teacher_flags_reference(seed, step, ids.cpu().numpy(), steps, p))
    f = teacher_forcing_flags(ids, 5, 0.3, 11, 3).cpu().numpy()
    perm = torch.randperm(ids.numel(), generator=torch.Generator().manual_seed(0))
    g = teacher_forcing_flags(ids[perm.cuda()], 5, 0.3, 11, 3).cpu().numpy()
    np.testing.assert_array_equal(g, f[:, perm.numpy()])   # a pure function of the sample, whatever its slot
    n = f.size
    assert abs(f.mean() - 0.3) <= 4 * np.sqrt(0.3 * 0.7 / n), f.mean()


# ------------------------------------------------------------------------------------------------ Fno2d.rollout
def _grads(m, bt, gseq, steps, noise=None, teacher=None):
    x = bt["inputs"].clone().requires_grad_(True)
    cp = bt["case_params"].clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    seq = m.rollout(x, cp, bt["mask"], steps, noise=noise, teacher=teacher)
    (seq * gseq).sum().backward()
    torch.cuda.synchronize()
    return seq.detach(), [p.grad.clone() for p in m.parameters()], x.grad, cp.grad


def _truth(bt, steps, seed):
    """true frames for steps 1 .. K-1, masked as rollout_batch's targets are"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    b, _, gh, gw = bt["inputs"].shape
    return torch.randn(steps - 1, b, 2, gh, gw, device="cuda", generator=g) * bt["mask"].view(1, b, 1, gh, gw)


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("config", list(WHERE))
@pytest.mark.parametrize("noisy", [False, True], ids=["plain", "noise"])
def test_zero_flags_are_the_rollout_without_teacher_bit_for_bit(config, K, noisy):
    where, act = WHERE[config]
    b = 5
    sd, bt, gseq = _case(60 + K, where, b, 5, K)
    m = _model(sd, 5, 4, act).cuda()
    noise = RolloutNoise(0.05, 3, 7, torch.arange(b, device="cuda") * 3) if noisy else None
    teacher = TeacherForcing(_truth(bt, K, 1), torch.zeros(K - 1, b, dtype=torch.uint8, device="cuda"))
    a = _grads(m, bt, gseq, K, noise=noise)
    t = _grads(m, bt, gseq, K, noise=noise, teacher=teacher)
    assert torch.equal(a[0], t[0])
    for (name, _), ga, gt in zip(m.named_parameters(), a[1], t[1]):
        assert torch.equal(ga, gt), name
    assert torch.equal(a[2], t[2]) and torch.equal(a[3], t[3])


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("config", list(WHERE))
def test_all_flags_feed_each_step_its_true_frame(config, K):
    where, act = WHERE[config]
    b = 4
    sd, bt, gseq = _case(70 + K, where, b, 5, K)
    m = _model(sd, 5, 4, act).cuda()
    truth = _truth(bt, K, 2)
    with torch.no_grad():
        seq = m.rollout(bt["inputs"], bt["case_params"], bt["mask"], K,
                        teacher=TeacherForcing(truth, torch.ones(K - 1, b, dtype=torch.bool, device="cuda")))
        for s in range(1, K):
            one = m.rollout(truth[s - 1], bt["case_params"], bt["mask"], 1)[0]
            assert torch.equal(seq[s], one), s


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("config", list(WHERE))
def test_mixed_flags_match_the_float64_oracle(config, K, request):
    where, act = WHERE[config]
    b, depth = 6, 4
    sd, bt, gseq = _case(80 + K, where, b, 5, K, depth)
    m = _model(sd, 5, depth, act).cuda()
    truth = _truth(bt, K, 3)
    flags = torch.tensor([[(s + i) % 2 for i in range(b)] for s in range(K - 1)], dtype=torch.uint8, device="cuda")
    seq, grads, d_in, d_cp = _grads(m, bt, gseq, K, teacher=TeacherForcing(truth, flags))
    # the same loss through chained one-step rollouts under autograd, the fed frame chosen with torch.where: the same
    # kernels on the same frames, so bit-identical predictions and gradients up to the summation order (CHAINED_BAR)
    x0 = bt["inputs"].clone().requires_grad_(True)
    cp = bt["case_params"].clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    x, preds = x0, []
    for s in range(K):
        if s > 0:
            x = torch.where(flags[s - 1].bool().view(-1, 1, 1, 1), truth[s - 1], x)
        x = m.rollout(x, cp, bt["mask"], 1)[0]
        preds.append(x)
    (torch.stack(preds) * gseq).sum().backward()
    assert torch.equal(torch.stack(preds).detach(), seq)
    chained = {k: _rel(g, p.grad) for (k, p), g in zip(m.named_parameters(), grads)}
    chained.update(d_inputs=_rel(d_in, x0.grad), d_case_params=_rel(d_cp, cp.grad))
    worst = max(chained, key=chained.get)
    assert chained[worst] <= CHAINED_BAR, (worst, chained[worst])
    if act == "float32":   # the float64 oracle linearised at the GPU's frames (the rollout tests' fp32 bars)
        f64 = lambda t: t.detach().cpu().to(torch.complex128 if t.is_complex() else torch.float64).numpy()
        ref, d_in_ref, d_cp_ref = teacher_rollout_vjp(sd, f64(bt["inputs"]), f64(bt["case_params"]), f64(bt["mask"]),
                                                      f64(gseq), f64(truth), flags.cpu().numpy(), frames=f64(seq))
        errs = {k: float(np.linalg.norm(f64(g) - ref[k]) / np.linalg.norm(ref[k]))
                for (k, _), g in zip(m.named_parameters(), grads)}
        worst = max(errs, key=errs.get)
        out = {"grad.max": errs[worst], "grad.worst": worst, "d_inputs": _max_rel(f64(d_in), d_in_ref),
               "d_case_params": _max_rel(f64(d_cp), d_cp_ref)}
        _report(request.node.callspec.id, out)
        fails = [(k, out[k]) for k in ("grad.max", "d_inputs", "d_case_params")
                 if not out[k] <= backward_bar(depth, K, k.split(".")[0])]
        assert not fails, fails
    # the forced samples' inputs are the true frames: their predictions equal one-step rollouts from them
    with torch.no_grad():
        for s in range(1, K):
            one = m.rollout(truth[s - 1], bt["case_params"], bt["mask"], 1)[0]
            fs = flags[s - 1].bool()
            assert torch.equal(seq[s][fs], one[fs]), s


@pytest.mark.parametrize("config", list(WHERE))
def test_a_nan_in_a_forced_sample_stays_out_of_its_next_input_and_carry(config):
    where, act = WHERE[config]
    b, K = 4, 2
    sd, bt, gseq = _case(90, where, b, 5, K)
    m = _model(sd, 5, 4, act).cuda()
    truth = _truth(bt, K, 4)
    flags = torch.tensor([[1, 0, 1, 0]], dtype=torch.uint8, device="cuda")
    # a NaN in sample 0's start frame: its prediction 0 is NaN, but step 1 is fed its true frame
    bt_nan = dict(bt, inputs=bt["inputs"].clone())
    bt_nan["inputs"][0, 0, 3, 5] = float("nan")
    seq, _, d_in, _ = _grads(m, bt_nan, gseq, K, teacher=TeacherForcing(truth, flags))
    assert torch.isnan(seq[0, 0]).any()
    assert torch.isfinite(seq[1]).all() and torch.isfinite(seq[:, 1:]).all()
    assert torch.isfinite(d_in[1:]).all()
    # a NaN in step 1's upstream gradient of sample 2 (so in its dL/da0): sample 2's carry into prediction 0 is
    # dpreds[0] alone, so its d_inputs are step 0's own, bit for bit; the other samples stay finite
    g_nan = gseq.clone()
    g_nan[1, 2, 1, 7, 9] = float("nan")
    seq2, _, d_in2, d_cp2 = _grads(m, bt, g_nan, K, teacher=TeacherForcing(truth, flags))
    own = _grads(m, bt, gseq[:1], 1)
    assert torch.equal(d_in2[2], own[2][2])
    keep = [0, 1, 3]
    assert torch.isfinite(d_in2[keep]).all() and torch.isfinite(d_cp2[keep]).all()


# ------------------------------------------------------------------------------------------------ train_auto
def _eager_loop(model, frames, windows, K, probs, teacher_seed, sigma, noise_seed, every, num_epochs, lr, lr_gamma,
                batch_size, eval_interval, generator, **opts):
    """The loop of train_auto's docstring (INTEGRATION §3) with FusedAdam(**opts), a real StepLR and the evaluation
    loader's RNG draw."""
    from cfdbench_b200.data import index_batches
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr, **opts)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=lr_gamma)
    losses, norms, t = [], [], 0
    for ep in range(num_epochs):
        for ib in index_batches(len(windows), batch_size, True, generator):
            t += 1
            b = frames.rollout_batch(windows[ib], K, noise_std=sigma, noise_seed=noise_seed, noise_step=t)
            ids = torch.as_tensor(windows[ib], device="cuda")
            flags = teacher_forcing_flags(ids, K, probs[ep], teacher_seed, t)
            noise = RolloutNoise(sigma, noise_seed, t, ids, 0) if every else None
            seq = model.rollout(b["inputs"], b["case_params"], b["mask"], K, noise=noise,
                                teacher=TeacherForcing(b["labels"][:K - 1], flags))
            loss = sum(model.loss_fn(preds=seq[k], labels=b["labels"][k])["nmse"] for k in range(K)) / K
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


def _graph_vs_eager(tmp_path, config, K, teacher_forcing, sigma=0.0, every=False, epochs=4, **opts):
    problem, act_dtype, lengths, batch_size = CONFIGS[config]
    eval_interval, noise_seed, teacher_seed, lr_gamma = 2, 2 ** 63 + 9, 2 ** 64 - 5, 0.9
    ds, dev = _ChainSplit(lengths, problem, s=1, seed=31), _AutoSplit(4, problem, seed=32)
    windows = rollout_windows(ds.case_ids, K, 1)
    assert len(windows) % batch_size != 0, "the split must leave a ragged last batch"
    probs = [float(teacher_forcing)] * epochs if np.isscalar(teacher_forcing) else list(teacher_forcing)
    ref_m, m = _auto_model(problem, act_dtype, seed=8), _auto_model(problem, act_dtype, seed=8)
    ref_losses, ref_norms, ref_opt = _eager_loop(ref_m, DeviceFrames(ds, device="cuda"), windows, K, probs,
                                                 teacher_seed, sigma, noise_seed, every, epochs, 1e-3, lr_gamma,
                                                 batch_size, eval_interval, torch.Generator().manual_seed(5), **opts)
    out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, lr_gamma=lr_gamma, batch_size=batch_size,
                     eval_batch_size=3, eval_interval=eval_interval, rollout_steps=K, input_noise_std=sigma,
                     noise_seed=noise_seed, noise_every_step=every, teacher_forcing=teacher_forcing,
                     teacher_seed=teacher_seed, generator=torch.Generator().manual_seed(5), **opts)
    losses, opt = out["train_losses"], out["optimizer"]
    steps = epochs * -(-len(windows) // batch_size)
    assert len(losses) == len(ref_losses) == steps
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


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_teacher_forcing_is_bit_identical_to_the_eager_loop(tmp_path, config, K):
    _graph_vs_eager(tmp_path / "c", config, K, 0.5)
    _graph_vs_eager(tmp_path / "s", config, K, [1.0, 0.6, 0.3, 0.0])


@pytest.mark.parametrize("config", list(CONFIGS))
def test_teacher_forcing_with_noise_on_every_step_is_bit_identical_to_the_eager_loop(tmp_path, config):
    _graph_vs_eager(tmp_path, config, 4, [0.9, 0.5, 0.5, 0.1], sigma=0.05, every=True)


def test_teacher_forcing_with_clipping_and_ema_is_bit_identical_to_the_eager_loop(tmp_path):
    _graph_vs_eager(tmp_path, "cavity-f32", 4, 0.4, sigma=0.05, every=True, max_grad_norm=0.02, ema_decay=0.99)


def test_teacher_forcing_syncs_once_per_epoch_and_costs_k_frames(tmp_path):
    m = _auto_model("cavity", act_dtype="bfloat16", seed=6)
    dev = DeviceFrames(_AutoSplit(4, "cavity", seed=1), device="cuda")
    tr = DeviceFrames(_ChainSplit((20, 24, 22), "cavity", seed=2), device="cuda")
    K, B = 4, 8

    def run(epochs, tf):
        return train_auto(m, tr, dev, tmp_path, num_epochs=epochs, batch_size=B, eval_interval=1000, rollout_steps=K,
                          teacher_forcing=tf)
    run(1, 0.5)
    counts = {e: len(_count_syncs(lambda: run(e, 0.5))) for e in (1, 3)}
    assert counts == {1: 2, 3: 4}   # the chain check, then one per epoch

    def rise(tf):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(2, tf)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    plain, forced = rise(None), rise(0.5)
    frame = B * 2 * 64 * 64 * 4
    print(f"peak rise: plain {plain} B, teacher forcing {forced} B ({(forced - plain) / frame:.2f} frames)")
    assert forced <= plain + K * frame + 2 ** 20


def test_resumed_teacher_forced_run_equals_the_straight_run(tmp_path):
    ds, dev = _ChainSplit((9, 12, 7), "cavity", s=1, seed=31), _ChainSplit((8, 6), "cavity", s=1, seed=32)

    def call(out, epochs, model_seed, rng_seed):
        m = _auto_model("cavity", "bfloat16", seed=model_seed)
        torch.manual_seed(rng_seed)
        return m, train_auto(m, ds, dev, out, num_epochs=epochs, lr=1e-3, batch_size=8, eval_batch_size=3,
                             eval_interval=2, log_interval=1000, rollout_steps=4, input_noise_std=0.05, noise_seed=77,
                             noise_every_step=True, max_grad_norm=0.02, ema_decay=0.99, dev_rollout_steps=2,
                             teacher_forcing=[1.0, 0.8, 0.6, 0.4, 0.2], teacher_seed=3, resumable=True)
    straight = call(tmp_path / "a", 5, 8, 5) + (tmp_path / "a",)
    m1, r1 = call(tmp_path / "b", 2, 8, 5)   # interrupted after the evaluation of epoch 1
    state = torch.load(tmp_path / "b" / resume.STATE_NAME, map_location="cpu", weights_only=True)
    assert state["epoch"] == 1 and state["config"]["teacher_forcing"] == [1.0, 0.8, 0.6, 0.4, 0.2]
    torch.rand(7)
    m2, r2 = call(tmp_path / "b", 5, 99, 1234)
    assert r2["start_epoch"] == 2
    _assert_same_run(straight, (m2, r2, tmp_path / "b"))


# ------------------------------------------------------------------------------------------------ accuracy record
def test_record_rollout_error_of_teacher_forcing(tmp_path):
    """One seeded run per mode in the protocol of test_record_rollout_error_of_each_training_mode: K = 4, the free
    rollout against scheduled sampling from p = 1 to p = 0, the 1-step and 20-step infer_multistep NMSE.  A record, not
    a ranking."""
    from cfdbench_b200 import infer_multistep
    tr, test = _Dynamics(6, 24, seed=1), _Dynamics(3, 22, seed=2)
    epochs = 8
    modes = {"K=4 free": dict(rollout_steps=4),
             "K=4 teacher 1->0": dict(rollout_steps=4, teacher_forcing=list(np.linspace(1.0, 0.0, epochs)))}
    for i, (name, kw) in enumerate(modes.items()):
        m = _auto_model("cavity", seed=5)
        train_auto(m, tr, test, tmp_path / str(i), num_epochs=epochs, batch_size=8, eval_interval=1000,
                   generator=torch.Generator().manual_seed(0), **kw)
        cps = [torch.tensor([0.1 * j for j in range(5)]) for _ in test.all_features]
        nmse = [r["nmse"] for r in infer_multistep(m, test.all_features, cps, infer_steps=20)]
        print(f"ACCURACY {name}: nmse step 1 {nmse[0]:.4g}, step 20 {nmse[-1]:.4g}, mean {np.mean(nmse):.4g}")
        assert np.all(np.isfinite(nmse))
