"""Noise on every rollout step on the GPU: `fno_add_input_noise_stream` against `fno_add_input_noise` and the host
restatement (test_rollout_noise_host.noise_stream_reference) on three grids; `Fno2d.rollout(noise=...)` against the
eager chain of one-step rollouts on frames perturbed with `add_input_noise`, predictions bit for bit and gradients under
autograd; `train_auto(noise_every_step=True)` bit for bit against the eager loop of its docstring; the path without
noise; the memory a noisy rollout step adds; and a record of the rollout error it gives."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from cfdbench_b200 import RolloutNoise, _lib, add_input_noise
from test_gpu_eval_auto import _AutoSplit, _model
from test_gpu_train_pushforward import _Dynamics
from test_gpu_train_rollout import _ChainSplit
from test_rollout_noise_host import noise_stream_reference

pytestmark = pytest.mark.gpu


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _frames(b, gh, gw, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(b, 2, gh, gw, device="cuda", generator=g)
    mask = (torch.rand(b, 1, gh, gw, device="cuda", generator=g) < 0.8).float()
    return x, mask


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("gh,gw", [(64, 64), (66, 65), (25, 127)])
def test_stream_noise_against_add_input_noise_and_the_host(gh, gw):
    lib = _lib.load()
    b, seed, step = 5, 0x1234_5678_9ABC, 2 ** 33 + 17
    x, mask = _frames(b, gh, gw, seed=gh)
    idx = torch.tensor([11, 0, 5, 5, 7], device="cuda")
    base = torch.tensor([step - 4], dtype=torch.int64, device="cuda")
    off = torch.tensor([4], dtype=torch.int32, device="cuda")

    def stream_noise(inp, out, k, std=0.5, m=mask):
        assert lib.fno_add_input_noise_stream(inp.data_ptr(), out.data_ptr(), m.data_ptr(), idx.data_ptr(), b, gh, gw, std,
                                              seed, base.data_ptr(), off.data_ptr(), k, _st()) == 0, lib.fno_last_error()
    ref = x.clone()
    assert lib.fno_add_input_noise(ref.data_ptr(), mask.data_ptr(), idx.data_ptr(), b, gh, gw, 0.5, seed, base.data_ptr(),
                                   off.data_ptr(), _st()) == 0
    # stream 0: fno_add_input_noise bit for bit, in place and out of place
    inplace = x.clone()
    stream_noise(inplace, inplace, 0)
    out = torch.full_like(x, float("nan"))
    x0 = x.clone()
    stream_noise(x, out, 0)
    assert torch.equal(inplace, ref) and torch.equal(out, ref) and torch.equal(x, x0)
    on = (mask != 0).expand_as(x)
    assert torch.equal(out[~on], x[~on])   # out = in where the mask is 0
    # a 4-byte aligned slice (the 64x64 path's scalar branch) gives the same frames
    buf = torch.zeros(b * 2 * gh * gw + 1, device="cuda")
    xs = buf[1:].view(b, 2, gh, gw)
    xs.copy_(x)
    stream_noise(xs, xs, 0)
    assert torch.equal(xs, ref)
    # streams 1..7: the host restatement, distinct from stream 0 and from each other, whatever the batch slot
    zero, ones = torch.zeros_like(x), torch.ones_like(mask)
    zs = []
    for k in range(8):
        z = torch.empty_like(x)
        stream_noise(zero, z, k, std=1.0, m=ones)
        zs.append(z)
        got = z.double().cpu().numpy()
        for s, j in enumerate(idx.tolist()):
            want = noise_stream_reference(seed, step, j, 2 * gh * gw, k).reshape(2, gh, gw)
            tol = 8 * 2.0 ** -23 * np.maximum(1.0, np.abs(want))
            assert np.all(np.abs(got[s] - want) <= tol), (k, j, float((np.abs(got[s] - want) / tol).max()))
        assert torch.equal(z[2], z[3])   # the same sample in two slots
        if k > 0:
            out_k = torch.empty_like(x)
            stream_noise(x, out_k, k)
            assert torch.equal(out_k[~on], x[~on])
            assert torch.allclose(out_k, x + 0.5 * z * mask, rtol=1e-6, atol=1e-6)   # fmaf(0.5 z, mask, x)
    for a in range(8):
        for c in range(a):
            assert not torch.any(zs[a][:3] == zs[c][:3]), (a, c)
    # the sample's index, not its slot: a permuted batch gives the permuted noise
    perm = torch.tensor([4, 2, 0, 1, 3], device="cuda")
    idx_p = idx[perm]
    zp = torch.empty_like(x)
    assert lib.fno_add_input_noise_stream(zero.data_ptr(), zp.data_ptr(), ones.data_ptr(), idx_p.data_ptr(), b, gh, gw, 1.0,
                                          seed, base.data_ptr(), off.data_ptr(), 3, _st()) == 0
    assert torch.equal(zp, zs[3][perm])


# ------------------------------------------------------------------------------------------------ Fno2d.rollout(noise)
ROLLOUT_CONFIGS = {"cavity-f32": ("cavity", "float32"), "cavity-bf16": ("cavity", "bfloat16"), "tube": ("tube", "float32")}


def _chain(m, x, cp, mk, K, noise):
    """The eager chain: K one-step rollouts, step s fed its predecessor perturbed with stream k0 + s (not stream 0)."""
    preds, cur = [], x
    for s in range(K):
        if noise.k0 + s > 0:
            cur = add_input_noise(cur, mk, noise.ids, noise.std, noise.seed, noise.step, stream=noise.k0 + s)
        cur = m.rollout(cur, cp, mk, 1)[0]
        preds.append(cur)
    return torch.stack(preds)


@pytest.mark.parametrize("K,B,k0", [(1, 1, 0), (2, 3, 0), (4, 3, 0), (3, 70, 1), (4, 1, 2), (1, 3, 3)])
@pytest.mark.parametrize("config", list(ROLLOUT_CONFIGS))
def test_rollout_noise_equals_the_eager_chain(config, K, B, k0):
    problem, act_dtype = ROLLOUT_CONFIGS[config]
    gh, gw = (66, 65) if problem == "tube" else (64, 64)
    m, ref = _model(problem, act_dtype, seed=4), _model(problem, act_dtype, seed=4)
    x, mk = _frames(B, gh, gw, seed=B + K)
    x = x * mk
    cp = torch.rand(B, m.n_case_params, device="cuda")
    ids = torch.randint(0, 10 ** 6, (B,), device="cuda")
    noise = RolloutNoise(0.05, 2 ** 63 + 3, 12345, ids, k0)
    w = torch.randn(K, B, 2, gh, gw, device="cuda")

    def run(model, fn):
        xi, ci = x.clone().requires_grad_(True), cp.clone().requires_grad_(True)
        seq = fn(model, xi, ci)
        (seq * w).sum().backward()
        grads = [p.grad.clone() for p in model.parameters()]
        model.zero_grad()
        return seq.detach(), grads, xi.grad, ci.grad
    seq, grads, dx, dcp = run(m, lambda mod, xi, ci: mod.rollout(xi, ci, mk, K, noise=noise))
    seq_r, grads_r, dx_r, dcp_r = run(ref, lambda mod, xi, ci: _chain(mod, xi, ci, mk, K, noise))
    assert torch.equal(seq, seq_r)

    def rel(a, b):
        return float((a - b).norm() / b.norm().clamp_min(1e-30))
    errs = [rel(a, b) for a, b in zip(grads, grads_r)] + [rel(dx, dx_r), rel(dcp, dcp_r)]
    print(f"{config} K={K} B={B} k0={k0}: max gradient rel err {max(errs):.2e}")
    assert max(errs) <= 1e-5
    # no autograd, direct launches and a repeated call (the graph's refilled step and ids) give the same predictions
    with torch.no_grad():
        assert torch.equal(m.rollout(x, cp, mk, K, noise=noise), seq)
        m.graph_rollout = False
        assert torch.equal(m.rollout(x, cp, mk, K, noise=noise), seq)
        m.graph_rollout = True
        other = m.rollout(x, cp, mk, K, noise=noise._replace(step=noise.step + 1))
        for s in range(K):
            assert torch.equal(other[s], seq[s]) == (k0 + s == 0), s   # only the noisy steps change
        assert torch.equal(m.rollout(x, cp, mk, K, noise=noise), seq)


def test_sweep_graph_is_reused_across_seeds_and_std():
    """The sweep reads only k0 and the fed frames: a new seed, std or step reuses its captured graph, and the gradients
    stay those of direct launches."""
    m, ref = _model("cavity", "float32", seed=4), _model("cavity", "float32", seed=4)
    ref.graph_rollout = False
    x, mk = _frames(3, 64, 64, seed=9)
    cp = torch.rand(3, m.n_case_params, device="cuda")
    ids = torch.tensor([4, 8, 15], device="cuda")
    w = torch.randn(3, 3, 2, 64, 64, device="cuda")
    for i, noise in enumerate((RolloutNoise(0.05, 1, 7, ids, 1), RolloutNoise(0.2, 99, 8, ids.flip(0), 1))):
        grads = []
        for model in (m, ref):
            xi = x.clone().requires_grad_(True)
            (model.rollout(xi, cp, mk, 3, noise=noise) * w).sum().backward()
            grads.append([p.grad.clone() for p in model.parameters()] + [xi.grad])
            model.zero_grad()
        assert all(torch.equal(a, b) for a, b in zip(*grads)), i
        assert sum(1 for k in m._train_graphs if k[0] == "bwd") == 1


def test_rollout_without_noise_is_todays_path(monkeypatch):
    """noise=None and std 0 issue the entry points and give the predictions of a rollout without the argument."""
    from cfdbench_b200 import fno2d
    m = _model("cavity", "bfloat16", seed=2)
    x, mk = _frames(3, 64, 64, seed=1)
    cp = torch.rand(3, m.n_case_params, device="cuda")
    ids = torch.arange(3, device="cuda")
    calls = []
    orig = fno2d._Route.call

    def record(self, name, *args):
        calls.append(name)
        return orig(self, name, *args)
    monkeypatch.setattr(fno2d._Route, "call", record)
    m.graph_rollout = False   # every call issues its entry points (a graph replay issues none)
    outs = []
    for noise in ("omitted", None, RolloutNoise(0.0, 1, 2, ids, 1)):
        calls.clear()
        xi = x.clone().requires_grad_(True)
        kw = {} if noise == "omitted" else dict(noise=noise)
        seq = m.rollout(xi, cp, mk, 3, **kw)
        seq.sum().backward()
        outs.append((seq.detach(), xi.grad, list(calls)))
    assert outs[0][2] == ["rollout_forward_train", "rollout_backward"]
    for seq, dx, names in outs[1:]:
        assert torch.equal(seq, outs[0][0]) and torch.equal(dx, outs[0][1]) and names == outs[0][2]


# ------------------------------------------------------------------------------------------------ train_auto
def _eager_every_step(model, frames, windows, K, G, sigma, noise_seed, num_epochs, lr, lr_gamma, batch_size,
                      eval_interval, generator):
    """The loop of train_auto's docstring for noise_every_step=True."""
    from cfdbench_b200 import FusedAdam
    from cfdbench_b200.data import index_batches
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=lr_gamma)
    losses, t = [], 0
    for ep in range(num_epochs):
        for ib in index_batches(len(windows), batch_size, True, generator):
            t += 1
            idx = windows[ib]
            b = frames.rollout_batch(idx, K, noise_std=sigma, noise_seed=noise_seed, noise_step=t)
            ids = torch.as_tensor(idx, device=b["inputs"].device)
            x = b["inputs"]
            for k in range(K - G):
                if k > 0:
                    x = add_input_noise(x, b["mask"], ids, sigma, noise_seed, t, stream=k)
                with torch.no_grad():
                    x = model.generate_many(x, b["case_params"], b["mask"], 1)[0]
            seq = model.rollout(x, b["case_params"], b["mask"], G, noise=RolloutNoise(sigma, noise_seed, t, ids, K - G))
            loss = sum(model.loss_fn(preds=seq[g], labels=b["labels"][K - G + g])["nmse"] for g in range(G)) / G
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss.item())
        sched.step()
        if (ep + 1) % eval_interval == 0:
            dev_eval_draw(generator)
    return losses, opt


TRAIN_CONFIGS = {  # problem, act_dtype, case lengths, batch_size
    "cavity-ragged": ("cavity", "float32", (9, 14, 7), 8),
    "cavity-bf16": ("cavity", "bfloat16", (12, 10), 4),
    "tube": ("tube", "float32", (9, 8, 10), 8),
}


@pytest.mark.parametrize("K,G", [(2, 1), (4, 1), (4, 2), (4, 4)])
@pytest.mark.parametrize("config", list(TRAIN_CONFIGS))
def test_train_auto_every_step_noise_is_bit_identical_to_the_eager_loop(tmp_path, config, K, G):
    from cfdbench_b200 import DeviceFrames, rollout_windows, train_auto
    problem, act_dtype, lengths, batch_size = TRAIN_CONFIGS[config]
    epochs, eval_interval, sigma, noise_seed = 3, 2, 0.05, 2 ** 63 + 9
    ds, dev = _ChainSplit(lengths, problem, s=1, seed=31), _AutoSplit(4, problem, seed=32)
    windows = rollout_windows(ds.case_ids, K, 1)
    ref_m, m = _model(problem, act_dtype, seed=8), _model(problem, act_dtype, seed=8)
    ref_losses, ref_opt = _eager_every_step(ref_m, DeviceFrames(ds, device="cuda"), windows, K, G, sigma, noise_seed,
                                            epochs, 1e-3, 0.9, batch_size, eval_interval,
                                            torch.Generator().manual_seed(5))
    out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, batch_size=batch_size, eval_batch_size=3,
                     eval_interval=eval_interval, rollout_steps=K, rollout_grad_steps=G, input_noise_std=sigma,
                     noise_seed=noise_seed, noise_every_step=True, generator=torch.Generator().manual_seed(5))
    losses, opt = out["train_losses"], out["optimizer"]
    assert len(losses) == len(ref_losses) == epochs * -(-len(windows) // batch_size)
    assert losses == ref_losses
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        sa, sb = opt.state[a], ref_opt.state[b]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
    # noise on the start frame only trains another model
    start_only = _model(problem, act_dtype, seed=8)
    train_auto(start_only, ds, dev, tmp_path / "start", num_epochs=epochs, lr=1e-3, batch_size=batch_size,
               eval_batch_size=3, eval_interval=eval_interval, rollout_steps=K, rollout_grad_steps=G, input_noise_std=sigma,
               noise_seed=noise_seed, generator=torch.Generator().manual_seed(5))
    assert any(not torch.equal(a, b) for a, b in zip(m.parameters(), start_only.parameters()))


@pytest.mark.parametrize("K", [1, 3])
def test_the_flag_without_effect_is_the_default_path(tmp_path, K):
    """K = 1 with the flag, and the flag without noise, train exactly as without it."""
    from cfdbench_b200 import train_auto
    ds, dev = _ChainSplit((11, 12), "cavity", seed=1), _AutoSplit(4, "cavity", seed=2)
    noise = dict(input_noise_std=0.05, noise_seed=5) if K == 1 else {}
    outs, models = [], []
    for i, every in enumerate((False, True)):
        m = _model("cavity", seed=3)
        outs.append(train_auto(m, ds, dev, tmp_path / str(i), num_epochs=2, batch_size=8, eval_interval=2,
                               rollout_steps=K, generator=torch.Generator().manual_seed(4), noise_every_step=every,
                               **noise))
        models.append(m)
    assert outs[0]["train_losses"] == outs[1]["train_losses"]
    for a, b in zip(models[0].parameters(), models[1].parameters()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("K,G", [(4, 1), (4, 4)])
def test_every_step_noise_adds_at_most_one_frame_per_step(K, G):
    """The peak memory of building a rollout step's graphs and training one epoch on them, with noise on every step
    against noise on the start frame: the fed-frame buffers, one frame per rollout step, and nothing else.  The peak is
    the caching allocator's peak of requested bytes: its allocated-bytes peak counts whole blocks, and a block can be
    larger than its request (a large-pool block whose remainder is 1 MiB or less is not split), so where the blocks
    fall shifts that peak by up to about a frame either way at B = 32 (a 1 MiB frame)."""
    from cfdbench_b200 import DeviceFrames, FusedAdam, rollout_windows
    from cfdbench_b200.train import _RolloutStepGraphs, epoch_permutation
    m = _model("cavity", act_dtype="bfloat16", seed=6)
    tr = DeviceFrames(_ChainSplit((40, 44, 42), "cavity", seed=2), device="cuda")
    windows = rollout_windows(tr._case_ids_host, K, 1)
    bs = 32

    def rise(every):
        gc.collect()
        torch.cuda.synchronize()
        base = torch.cuda.memory_stats()["requested_bytes.all.current"]
        base_blocks = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        graphs = _RolloutStepGraphs(m, tr, bs, FusedAdam(m.parameters(), lr=1e-3), windows.size, K, 1, G,
                                    noise_std=0.01, noise_seed=1, noise_every_step=every)
        graphs.epoch(windows[epoch_permutation(windows.size, bs, torch.Generator().manual_seed(0))], 1e-3, 1)
        torch.cuda.synchronize()
        peak = torch.cuda.memory_stats()["requested_bytes.all.peak"] - base
        peak_blocks = torch.cuda.max_memory_allocated() - base_blocks
        io = {k: (tuple(t.shape), t.dtype) for k, t in graphs.io.items() if isinstance(t, torch.Tensor)}
        del graphs
        return peak, peak_blocks, io
    rise(False)   # warm the model's caches
    (r0, b0, io0), (r1, b1, io1) = rise(False), rise(True)
    frame = bs * 2 * 64 * 64 * 4
    print(f"K={K} G={G} B={bs}: requested-bytes peak rise {r0} B start-only, {r1} B every step, "
          f"{(r1 - r0) / frame:.4f} frames; allocated-blocks peak {(b1 - b0) / frame:.3f} frames")
    # the step's buffers: the same, plus the fed frames of the trained steps and of the prefix, K frames in all
    extra = {k: v for k, v in io1.items() if k not in io0}
    assert {k: v for k, v in io1.items() if k in io0} == io0
    assert sorted(extra) == sorted(["fed"] + (["fed_prefix"] if G < K else []))
    assert sum(v[0][0] for v in extra.values()) == K and all(v[0][1:] == (bs, 2, 64, 64) for v in extra.values())
    assert r1 - r0 <= K * frame


# ------------------------------------------------------------------------------------------------ accuracy record
def test_record_rollout_error_with_every_step_noise(tmp_path):
    """The protocol of test_record_rollout_error_of_each_training_mode (one seeded run per mode, 8 epochs, the 20-step
    infer_multistep NMSE), for pushforward and full rollouts with noise on the start frame and on every step.  A record,
    not a ranking."""
    from cfdbench_b200 import infer_multistep, train_auto
    tr, test = _Dynamics(6, 24, seed=1), _Dynamics(3, 22, seed=2)
    noise = dict(input_noise_std=0.01, noise_seed=1)
    modes = {"K=4 G=1 noise 0.01 start": dict(rollout_steps=4, rollout_grad_steps=1, **noise),
             "K=4 G=1 noise 0.01 every step": dict(rollout_steps=4, rollout_grad_steps=1, noise_every_step=True, **noise),
             "K=4 G=4 noise 0.01 start": dict(rollout_steps=4, **noise),
             "K=4 G=4 noise 0.01 every step": dict(rollout_steps=4, noise_every_step=True, **noise)}
    for i, (name, kw) in enumerate(modes.items()):
        m = _model("cavity", seed=5)
        train_auto(m, tr, test, tmp_path / str(i), num_epochs=8, batch_size=8, eval_interval=1000,
                   generator=torch.Generator().manual_seed(0), **kw)
        cps = [torch.tensor([0.1 * j for j in range(5)]) for _ in test.all_features]
        nmse = [r["nmse"] for r in infer_multistep(m, test.all_features, cps, infer_steps=20)]
        print(f"ACCURACY {name}: nmse step 1 {nmse[0]:.4g}, step 20 {nmse[-1]:.4g}, mean {np.mean(nmse):.4g}")
        assert np.all(np.isfinite(nmse))
