"""Training noise and pushforward training on the GPU: `fno_add_input_noise` against the host restatement
(test_train_noise_host.noise_reference) on three grids, its reproducibility across calls, graph replays and batch
slots, its statistics; `train_auto(input_noise_std=..., rollout_grad_steps=...)` bit for bit against the eager loop
a user writes with `DeviceFrames.rollout_batch(noise_...)` + `generate_many` + `Fno2d.rollout`; the explicit defaults;
one synchronisation per epoch, flat memory; and a record of the rollout error each training mode gives."""
import ctypes as C

import numpy as np
import pytest
import torch

from cfdbench_b200 import _lib
from test_gpu_eval_auto import _AutoSplit, _model
from test_gpu_train_rollout import _ChainSplit, _count_syncs
from test_train_noise_host import noise_reference

pytestmark = pytest.mark.gpu


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class _ZeroSplit:
    """n samples on a gh x gw grid: zero velocity channels and a random 0/1 mask."""

    def __init__(self, n, gh, gw, seed=0):
        rng = np.random.default_rng(seed)
        fr = np.zeros((n, 3, gh, gw), np.float32)
        fr[:, 2] = rng.random((n, gh, gw)) < 0.8
        self.inputs, self.labels = torch.from_numpy(fr), torch.from_numpy(fr.copy())
        self.case_ids = np.arange(n) // 3
        self.case_params = [{"p0": 0.5 * c} for c in range(self.case_ids[-1] + 1)]


def _noise(z_got, mask):
    """float64 noise and the mask, per sample, from a batch of zero inputs (b, 2, h, w) and masks (b, 1, h, w)."""
    return z_got.double().cpu().numpy(), np.broadcast_to(mask.cpu().numpy(), z_got.shape)


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("gh,gw", [(64, 64), (66, 65), (25, 127)])
@pytest.mark.parametrize("frame_dtype", [torch.float32, torch.bfloat16])
def test_noise_matches_the_host_restatement(gh, gw, frame_dtype):
    from cfdbench_b200 import DeviceFrames
    fr = DeviceFrames(_ZeroSplit(12, gh, gw, seed=gh), device="cuda", frame_dtype=frame_dtype)
    idx = [11, 0, 5, 5, 7]
    seed, step = 0x1234_5678_9ABC, 2 ** 33 + 17
    b = fr.batch(idx, noise_std=1.0, noise_seed=seed, noise_step=step)
    got, mask = _noise(b["inputs"], b["mask"])
    n_el = 2 * gh * gw
    for s, j in enumerate(idx):
        z = noise_reference(seed, step, j, n_el).reshape(2, gh, gw)
        on = mask[s] != 0
        tol = 8 * 2.0 ** -23 * np.maximum(1.0, np.abs(z))
        err = np.abs(got[s] - z)
        assert np.all(err[on] <= tol[on]), (j, float((err / tol)[on].max()))
        assert np.all(got[s][~on] == 0) and not np.any(np.signbit(got[s][~on]))   # bit-identical to the input 0.0
        assert on.any() and (~on).any()
    assert torch.equal(b["inputs"][2], b["inputs"][3])   # the same sample in two slots
    ref = fr.batch(idx)
    for k in ("label", "mask", "case_params"):
        assert torch.equal(b[k], ref[k]), k   # only the inputs are perturbed
    # the raw entry point on a 4-byte aligned slice (the 64x64 path's scalar branch) and a scalar std
    x = torch.zeros(5 * 2 * gh * gw + 1, device="cuda")
    mk = torch.zeros(5 * gh * gw + 1, device="cuda")
    xv, mv = x[1:].view(5, 2, gh, gw), mk[1:].view(5, 1, gh, gw)
    mv.copy_(b["mask"])
    idx_d = torch.tensor(idx, device="cuda")
    base = torch.tensor([step - 4], dtype=torch.int64, device="cuda")
    off = torch.tensor([4], dtype=torch.int32, device="cuda")
    assert _lib.load().fno_add_input_noise(xv.data_ptr(), mv.data_ptr(), idx_d.data_ptr(), 5, gh, gw, 0.5, seed,
                                           base.data_ptr(), off.data_ptr(), _st()) == 0
    assert x[0] == 0
    assert torch.equal(xv, (b["inputs"] * 0.5)), "std * z: the step is base + offset, alignment does not matter"


def test_noise_is_reproducible_and_keyed_on_seed_step_and_sample():
    from cfdbench_b200 import DeviceFrames
    fr = DeviceFrames(_ZeroSplit(9, 66, 65, seed=1), device="cuda")
    kw = dict(noise_std=1.0, noise_seed=3, noise_step=5)
    a = fr.batch([1, 2, 3], **kw)["inputs"]
    assert torch.equal(a, fr.batch([1, 2, 3], **kw)["inputs"])
    c = fr.batch([3, 8, 1], **kw)["inputs"]   # batch composition and slot do not matter
    assert torch.equal(c[0], a[2]) and torch.equal(c[2], a[0])
    m = fr.batch([1], **kw)["mask"][0].expand(2, -1, -1) != 0
    for other in (dict(noise_seed=4), dict(noise_seed=3 + 2 ** 32), dict(noise_step=6), dict(noise_step=5 + 2 ** 32)):
        d = fr.batch([1, 2, 3], **{**kw, **other})["inputs"]
        assert not torch.any(d[0][m] == a[0][m]), other
    assert not torch.any(a[0][m] == a[1][m])   # another sample, another stream
    # rollout_batch perturbs the start inputs only, with the same noise
    rb = fr.rollout_batch([0, 1, 3, 4], 2, time_step_size=1, **kw)   # windows inside the cases of 3 samples
    assert torch.equal(rb["inputs"], fr.batch([0, 1, 3, 4], **kw)["inputs"])
    assert torch.equal(rb["labels"], fr.rollout_batch([0, 1, 3, 4], 2, 1)["labels"])
    # graph replay: the step is read when the kernel runs
    lib = _lib.load()
    x = torch.zeros(3, 2, 66, 65, device="cuda")
    mk = fr.batch([1, 2, 3])["mask"]
    idx = torch.tensor([1, 2, 3], device="cuda")
    base = torch.zeros(1, dtype=torch.int64, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        g.capture_begin(capture_error_mode="thread_local")
        try:
            assert lib.fno_add_input_noise(x.data_ptr(), mk.data_ptr(), idx.data_ptr(), 3, 66, 65, 1.0, 3,
                                           base.data_ptr(), off.data_ptr(), _st()) == 0
        finally:
            g.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    for b0, o in ((5, 0), (2, 3), (6, -1), (100, 7)):
        base.fill_(b0)
        off.fill_(o)
        x.zero_()
        g.replay()
        assert torch.equal(x, fr.batch([1, 2, 3], noise_std=1.0, noise_seed=3, noise_step=b0 + o)["inputs"]), (b0, o)


def test_noise_statistics():
    from cfdbench_b200 import DeviceFrames
    ds = _ZeroSplit(130, 64, 64, seed=2)
    ds.inputs[:, 2] = 1.0
    fr = DeviceFrames(ds, device="cuda")
    z = fr.batch(np.arange(128), noise_std=1.0, noise_seed=11, noise_step=1)["inputs"].double()
    n = z.numel()
    assert n >= 10 ** 6
    mean, var = float(z.mean()), float(z.var())
    print(f"{n} draws: mean {mean:.3e}, variance {var:.6f}")
    assert abs(mean) <= 6 / np.sqrt(n) and abs(var - 1) <= 6 * np.sqrt(2 / n)
    assert np.isclose(float((z.abs() < 1).double().mean()), 0.682689, atol=6 * np.sqrt(0.22 / n))


# ------------------------------------------------------------------------------------------------ against the eager loop
def _eager_loop(model, frames, windows, K, G, sigma, noise_seed, num_epochs, lr, lr_gamma, batch_size, eval_interval,
                generator):
    """The loop of train_auto's docstring, with FusedAdam, a real StepLR and the evaluation loader's RNG draw."""
    from cfdbench_b200 import FusedAdam
    from cfdbench_b200.data import index_batches
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=lr_gamma)
    losses, t = [], 0
    for ep in range(num_epochs):
        for ib in index_batches(len(windows), batch_size, True, generator):
            t += 1
            noise = dict(noise_std=sigma, noise_seed=noise_seed, noise_step=t)
            if K == 1:
                loss = model(**frames.batch(windows[ib], **noise))["loss"]["nmse"]
            else:
                b = frames.rollout_batch(windows[ib], K, **noise)
                x = b["inputs"]
                if K > G:
                    with torch.no_grad():
                        x = model.generate_many(x, b["case_params"], b["mask"], K - G)[-1]
                seq = model.rollout(x, b["case_params"], b["mask"], G)
                loss = sum(model.loss_fn(preds=seq[g], labels=b["labels"][K - G + g])["nmse"] for g in range(G)) / G
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss.item())
        sched.step()
        if (ep + 1) % eval_interval == 0:
            dev_eval_draw(generator)
    return losses, opt


CONFIGS = {  # problem, act_dtype, case lengths, batch_size, lr_gamma, frozen
    "cavity-ragged": ("cavity", "float32", (9, 14, 7), 8, 0.5, False),
    "cavity-bf16": ("cavity", "bfloat16", (12, 10), 4, 0.9, False),
    "cavity-b1": ("cavity", "float32", (6, 7), 1, 0.9, False),
    "cylinder": ("cylinder", "float32", (10, 11), 8, 0.9, False),
    "tube": ("tube", "float32", (9, 8, 10), 8, 0.9, False),
    "cavity-frozen": ("cavity", "float32", (10, 12), 8, 0.9, True),
}
FROZEN = ("fc0.weight", "blocks.1.conv0.weights2", "blocks.2.w0.bias", "fc2.bias")


@pytest.mark.parametrize("K,G,sigma", [(1, 1, 0.05), (2, 1, 0.0), (2, 1, 0.05), (4, 1, 0.0), (4, 1, 0.05), (4, 2, 0.0),
                                       (4, 2, 0.05), (4, 4, 0.05)])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_train_auto_noise_and_pushforward_are_bit_identical_to_the_eager_loop(tmp_path, config, K, G, sigma):
    from cfdbench_b200 import DeviceFrames, rollout_windows, train_auto
    problem, act_dtype, lengths, batch_size, lr_gamma, frozen = CONFIGS[config]
    epochs, eval_interval, noise_seed = 3, 2, 2 ** 63 + 9
    ds, dev = _ChainSplit(lengths, problem, s=1, seed=31), _AutoSplit(4, problem, seed=32)
    windows = rollout_windows(ds.case_ids, K, 1)
    ref_m, m = _model(problem, act_dtype, seed=8), _model(problem, act_dtype, seed=8)
    if frozen:
        for model in (ref_m, m):
            for name, prm in model.named_parameters():
                prm.requires_grad_(name not in FROZEN)
    ref_losses, ref_opt = _eager_loop(ref_m, DeviceFrames(ds, device="cuda"), windows, K, G, sigma, noise_seed, epochs,
                                      1e-3, lr_gamma, batch_size, eval_interval, torch.Generator().manual_seed(5))
    out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, lr_gamma=lr_gamma, batch_size=batch_size,
                     eval_batch_size=3, eval_interval=eval_interval, rollout_steps=K, rollout_grad_steps=G,
                     input_noise_std=sigma, noise_seed=noise_seed, generator=torch.Generator().manual_seed(5))
    losses, opt = out["train_losses"], out["optimizer"]
    steps = -(-len(windows) // batch_size)
    assert len(losses) == len(ref_losses) == epochs * steps
    print(f"{config} K={K} G={G} sigma={sigma}: max |loss diff| {max(abs(a - b) for a, b in zip(losses, ref_losses)):.3e}")
    assert losses == ref_losses
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        if frozen and name in FROZEN:
            assert a not in opt.state, name
            continue
        sa, sb = opt.state[a], ref_opt.state[b]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]), name
        assert torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert torch.equal(sa["step"], sb["step"]) and float(sa["step"]) == epochs * steps
    assert opt.param_groups[0]["lr"] == ref_opt.param_groups[0]["lr"]


@pytest.mark.parametrize("K", [1, 3])
def test_explicit_defaults_are_the_default_path(tmp_path, K):
    from cfdbench_b200 import train_auto
    ds, dev = _ChainSplit((11, 12), "cavity", seed=1), _AutoSplit(4, "cavity", seed=2)
    outs, models = [], []
    for i, kw in enumerate(({}, dict(input_noise_std=0.0, noise_seed=5, rollout_grad_steps=K))):
        m = _model("cavity", seed=3)
        outs.append(train_auto(m, ds, dev, tmp_path / str(i), num_epochs=3, batch_size=8, eval_interval=2,
                               rollout_steps=K, generator=torch.Generator().manual_seed(4), **kw))
        models.append(m)
    assert outs[0]["train_losses"] == outs[1]["train_losses"]
    for a, b in zip(models[0].parameters(), models[1].parameters()):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ syncs, memory
@pytest.mark.parametrize("K,G", [(1, 1), (4, 1)])
def test_noise_and_pushforward_syncs_and_memory(tmp_path, K, G):
    from cfdbench_b200 import DeviceFrames, train_auto
    m = _model("cavity", act_dtype="bfloat16", seed=6)
    dev = DeviceFrames(_AutoSplit(4, "cavity", seed=1), device="cuda")
    tr = DeviceFrames(_ChainSplit((20, 24, 22), "cavity", seed=2), device="cuda")

    def run(epochs):
        return train_auto(m, tr, dev, tmp_path, num_epochs=epochs, batch_size=8, eval_interval=1000, rollout_steps=K,
                          rollout_grad_steps=G, input_noise_std=0.01, noise_seed=1)
    run(1)
    counts = {e: len(_count_syncs(lambda: run(e))) for e in (1, 3)}
    chain = 1 if K > 1 else 0   # the chain check
    assert counts == {1: 1 + chain, 3: 3 + chain}

    def rise(epochs):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(epochs)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    r2, r6 = rise(2), rise(6)
    print(f"K={K} G={G}: peak rise 2 epochs {r2} B, 6 epochs {r6} B")
    assert r6 <= r2 + 4096


# ------------------------------------------------------------------------------------------------ accuracy record
class _Dynamics(_ChainSplit):
    """A linear, learnable evolution: each Fourier mode of a smooth field decays at its own rate per step."""

    def __init__(self, n_cases, t, seed=0):
        rng = np.random.default_rng(seed)
        x = np.linspace(0, 2 * np.pi, 64, dtype=np.float32)
        rates = {1: 0.97, 2: 0.9, 3: 0.8}
        cases = []
        for _ in range(n_cases):
            amp = {k: rng.standard_normal((2, 1, 1)).astype(np.float32) / k for k in rates}
            fr = np.zeros((t, 3, 64, 64), np.float32)
            for step in range(t):
                for k, r in rates.items():
                    fr[step, :2] += amp[k] * r ** step * np.sin(k * x)[:, None] * np.cos(k * x)[None, :]
            fr[:, 2] = 1.0
            cases.append(fr)
        self.all_features = [torch.from_numpy(c) for c in cases]
        self.inputs = torch.from_numpy(np.concatenate([c[:-1] for c in cases]))
        self.labels = torch.from_numpy(np.concatenate([c[1:] for c in cases]))
        self.case_ids = np.repeat(np.arange(n_cases), t - 1)
        self.time_step_size = 1
        self.case_params = [{f"p{j}": 0.1 * j for j in range(5)} for _ in range(n_cases)]


def test_record_rollout_error_of_each_training_mode(tmp_path):
    """One seeded run per mode, 8 epochs each: the 1-step and 20-step infer_multistep NMSE.  A record, not a ranking."""
    from cfdbench_b200 import infer_multistep, train_auto
    tr, test = _Dynamics(6, 24, seed=1), _Dynamics(3, 22, seed=2)
    modes = {"K=1": dict(), "K=1 noise 0.01": dict(input_noise_std=0.01, noise_seed=1),
             "K=4 G=1": dict(rollout_steps=4, rollout_grad_steps=1), "K=4 G=4": dict(rollout_steps=4)}
    for i, (name, kw) in enumerate(modes.items()):
        m = _model("cavity", seed=5)
        train_auto(m, tr, test, tmp_path / str(i), num_epochs=8, batch_size=8, eval_interval=1000,
                   generator=torch.Generator().manual_seed(0), **kw)
        cps = [torch.tensor([0.1 * j for j in range(5)]) for _ in test.all_features]
        nmse = [r["nmse"] for r in infer_multistep(m, test.all_features, cps, infer_steps=20)]
        print(f"ACCURACY {name}: nmse step 1 {nmse[0]:.4g}, step 20 {nmse[-1]:.4g}, mean {np.mean(nmse):.4g}")
        assert np.all(np.isfinite(nmse))
