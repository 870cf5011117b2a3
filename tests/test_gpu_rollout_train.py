"""`Fno2d.rollout`: training through a K-step rollout with one reused set of saved activations (fno_rollout_forward_train
+ the recomputing backward sweep fno_rollout_backward; fno_grid_* on other grids).

It must predict what K chained `generate` calls under autograd predict, bit for bit; give their gradients up to
summation order; match the float64 backpropagation through time (`oracle.fno_rollout_numpy.fno_rollout_vjp`) linearised
at the GPU's own frames; and keep its memory flat in K.  Every check prints its measured value (`-s`) before asserting."""
import json
import os

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle.fno_rollout_numpy import fno_rollout_vjp

pytestmark = pytest.mark.gpu


def _model(sd, p, depth, act):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=depth, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m


def _case(seed, where, b, p, steps, depth=4):
    """state dict, GPU batch (inputs, case_params, mask) and a random upstream gradient of the (K, B, 2, H, W) rollout"""
    sd = synth.make_state_dict(seed, n_params=p, depth=depth, spectral_gain=50.0)
    bt = synth.make_batch(seed + 1, b, where, with_label=False)
    rng = np.random.default_rng(seed + 2)
    if bt["case_params"].shape[1] != p:
        bt["case_params"] = rng.standard_normal((b, p)).astype(np.float32)
    gh, gw = bt["inputs"].shape[-2:]
    gseq = rng.standard_normal((steps, b, 2, gh, gw)).astype(np.float32)
    return sd, {k: torch.from_numpy(v).cuda() for k, v in bt.items()}, torch.from_numpy(gseq).cuda()


def _rollout_grads(m, bt, gseq, steps):
    """rollout + backward of sum(seq * gseq): (seq, parameter grads, d_inputs, d_case_params)"""
    x = bt["inputs"].clone().requires_grad_(True)
    cp = bt["case_params"].clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    seq = m.rollout(x, cp, bt["mask"], steps)
    (seq * gseq).sum().backward()
    torch.cuda.synchronize()
    return seq.detach(), [p.grad.clone() for p in m.parameters()], x.grad, cp.grad


def _chained_grads(m, bt, gseq, steps):
    """the same loss through `steps` chained `generate` calls under autograd"""
    x0 = bt["inputs"].clone().requires_grad_(True)
    cp = bt["case_params"].clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    x, preds = x0, []
    for s in range(steps):
        x = m.generate(x, cp, bt["mask"])
        preds.append(x)
    seq = torch.stack(preds)
    (seq * gseq).sum().backward()
    torch.cuda.synchronize()
    return seq.detach(), [p.grad.clone() for p in m.parameters()], x0.grad, cp.grad


def _rel(a, ref):
    a, ref = a.detach().double(), ref.detach().double()
    if a.is_complex():
        a, ref = torch.view_as_real(a), torch.view_as_real(ref)
    return float((a - ref).norm() / ref.norm())


def _max_rel(got, ref):
    """max over samples (axis 0) of the relative L2 error, float64 numpy"""
    b = ref.shape[0]
    d = np.linalg.norm((got - ref).reshape(b, -1), axis=1)
    return float(np.max(d / np.linalg.norm(ref.reshape(b, -1), axis=1)))


def _report(what, errs):
    print(f"\n[{what}] " + json.dumps({k: (float(f"{v:.3g}") if isinstance(v, float) else v) for k, v in errs.items()}))


# grid, storage, K, B, p
CONFIGS = [
    pytest.param("cavity", "float32", 8, 3, 5, id="64x64-fp32-K8-B3"),
    pytest.param("cavity", "bfloat16", 8, 3, 5, id="64x64-bf16-K8-B3"),
    pytest.param("cavity", "bfloat16", 3, 1, 5, id="64x64-bf16-K3-B1"),
    pytest.param("cylinder", "bfloat16", 4, 70, 8, id="64x64-bf16-K4-B70-holed"),
    pytest.param("cylinder", "float32", 2, 70, 8, id="64x64-fp32-K2-B70-holed"),
    pytest.param("tube", "float32", 5, 3, 5, id="66x65-fp32-K5-B3"),
    pytest.param("tube", "float32", 8, 1, 5, id="66x65-fp32-K8-B1"),
    pytest.param("tube", "float32", 3, 70, 5, id="66x65-fp32-K3-B70"),
]
# Gradients against chained `generate`: both backwards apply the same kernels to the same saved tensors and the same
# upstream gradients; the rollout adds each step's parameter gradients (and the project stage's batch chunks) straight
# into one buffer where autograd first reduces a step and then adds it, so only the summation order of K * chunks
# fp32 partial sums differs.
CHAINED_BAR = 1e-5


@pytest.mark.parametrize("where,act,steps,b,p", CONFIGS)
def test_rollout_equals_chained_generate(where, act, steps, b, p, request):
    sd, bt, gseq = _case(300 + steps * 7 + b, where, b, p, steps)
    m = _model(sd, p, 4, act)
    seq_r, g_r, din_r, dcp_r = _rollout_grads(m, bt, gseq, steps)
    seq_c, g_c, din_c, dcp_c = _chained_grads(m, bt, gseq, steps)
    assert seq_r.shape == (steps, b, 2) + tuple(bt["inputs"].shape[-2:]) and seq_r.dtype == torch.float32
    assert torch.equal(seq_r, seq_c), "predictions differ from chained generate"
    errs = {k: _rel(a, c) for (k, _), a, c in zip(m.named_parameters(), g_r, g_c)}
    worst = max(errs, key=errs.get)
    out = {"grad.max": errs[worst], "grad.worst": worst, "d_inputs": _rel(din_r, din_c),
           "d_case_params": _rel(dcp_r, dcp_c)}
    _report(request.node.callspec.id, out)
    assert errs[worst] <= CHAINED_BAR, (worst, errs[worst])
    assert out["d_inputs"] <= CHAINED_BAR and out["d_case_params"] <= CHAINED_BAR, out


def backward_bar(depth: int, steps: int, what: str) -> float:
    """Relative L2 bar against the float64 adjoint linearised at the GPU's frames.  One step's backward has the bar of
    test_gpu_train_conditioned (2.5e-6 per Fourier block plus projection and lift, twice that for d_case_params).  The
    rollout's gradient of step s's input passes through the backwards of steps s .. K-1, each adding its own fp32 error
    to the carry it hands on, and the parameter gradients are sums over the steps of such terms: the errors add up over
    at most K step backwards, so the bar is K times the single-step bar (DESIGN.md 5)."""
    return steps * (2.0 if what == "d_case_params" else 1.0) * 2.5e-6 * (depth + 1)


@pytest.mark.parametrize("where,steps,b,p", [
    pytest.param("cavity", 4, 3, 5, id="64x64-fp32-K4-B3"),
    pytest.param("cylinder", 3, 33, 8, id="64x64-fp32-K3-B33-holed"),
    pytest.param("tube", 4, 3, 5, id="66x65-fp32-K4-B3"),
])
def test_rollout_gradients_against_float64_bptt_at_the_gpu_frames(where, steps, b, p, request):
    depth = 4
    sd, bt, gseq = _case(500 + b, where, b, p, steps, depth)
    m = _model(sd, p, depth, "float32")
    seq, grads, d_in, d_cp = _rollout_grads(m, bt, gseq, steps)
    f64 = lambda t: t.detach().cpu().double().numpy() if not t.is_complex() else t.detach().cpu().to(torch.complex128).numpy()
    ref, d_in_ref, d_cp_ref = fno_rollout_vjp(sd, f64(bt["inputs"]), f64(bt["case_params"]), f64(bt["mask"]), f64(gseq),
                                              frames=f64(seq))
    errs, fails = {}, []
    for (k, _), g in zip(m.named_parameters(), grads):
        e = float(np.linalg.norm(f64(g) - ref[k]) / np.linalg.norm(ref[k]))
        errs[k] = e
    worst = max(errs, key=errs.get)
    out = {"grad.max": errs[worst], "grad.worst": worst, "d_inputs": _max_rel(f64(d_in), d_in_ref),
           "d_case_params": _max_rel(f64(d_cp), d_cp_ref)}
    bars = {"grad.max": backward_bar(depth, steps, "grad"), "d_inputs": backward_bar(depth, steps, "d_inputs"),
            "d_case_params": backward_bar(depth, steps, "d_case_params")}
    out["bars"] = {k: float(f"{v:.3g}") for k, v in bars.items()}
    _report(request.node.callspec.id, out)
    for k, bar in bars.items():
        if not out[k] <= bar:
            fails.append((k, out[k], bar))
    assert not fails, fails


@pytest.mark.parametrize("where,act", [("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32")])
def test_one_step_rollout_is_forward_plus_backward_bit_for_bit(where, act):
    sd, bt, gseq = _case(41, where, 33, 5, 1)
    m = _model(sd, 5, 4, act)
    seq, g_r, din_r, dcp_r = _rollout_grads(m, bt, gseq, 1)
    x = bt["inputs"].clone().requires_grad_(True)
    cp = bt["case_params"].clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    preds = m(inputs=x, case_params=cp, mask=bt["mask"])["preds"]
    (preds * gseq[0]).sum().backward()
    assert torch.equal(seq[0], preds.detach())
    for (k, prm), g in zip(m.named_parameters(), g_r):
        assert torch.equal(prm.grad, g), k
    assert torch.equal(x.grad, din_r) and torch.equal(cp.grad, dcp_r)


@pytest.mark.parametrize("where,act", [("cavity", "bfloat16"), ("tube", "float32")])
def test_repeated_sweeps_and_graph_vs_direct_launch_are_bit_identical(where, act):
    steps = 4
    sd, bt, gseq = _case(51, where, 5, 5, steps)
    m = _model(sd, 5, 4, act)
    assert m.graph_rollout
    runs = [_rollout_grads(m, bt, gseq, steps) for _ in range(3)]   # capture, then two replays
    m.graph_rollout = False
    runs.append(_rollout_grads(m, bt, gseq, steps))
    for r in runs[1:]:
        assert torch.equal(r[0], runs[0][0])
        for a, c in zip(r[1], runs[0][1]):
            assert torch.equal(a, c)
        assert torch.equal(r[2], runs[0][2]) and torch.equal(r[3], runs[0][3])


def test_graphs_follow_optimizer_steps():
    """A captured rollout graph reads its own copies of the packed weights: after an optimizer step it must compute
    with the new weights (graph replay == direct launch)."""
    from cfdbench_b200 import FusedAdam
    steps = 3
    sd, bt, gseq = _case(61, "cavity", 4, 5, steps)
    m = _model(sd, 5, 4, "bfloat16")
    opt = FusedAdam(m.parameters(), lr=1e-3)
    _rollout_grads(m, bt, gseq, steps)
    opt.step()
    got = _rollout_grads(m, bt, gseq, steps)
    m.graph_rollout = False
    ref = _rollout_grads(m, bt, gseq, steps)
    assert torch.equal(got[0], ref[0])
    for a, c in zip(got[1], ref[1]):
        assert torch.equal(a, c)


@pytest.mark.parametrize("where,act", [("cavity", "bfloat16"), ("tube", "float32")])
def test_no_grad_rollout_returns_the_same_predictions_without_a_graph(where, act):
    steps = 3
    sd, bt, gseq = _case(71, where, 3, 5, steps)
    m = _model(sd, 5, 4, act)
    seq, *_ = _rollout_grads(m, bt, gseq, steps)
    with torch.no_grad():
        ng = m.rollout(bt["inputs"], bt["case_params"], bt["mask"], steps)
    assert ng.grad_fn is None and not ng.requires_grad
    assert torch.equal(ng, seq)
    # unbatched (c,h,w) / (p,) / (h,w) arguments get a batch axis
    with torch.no_grad():
        one = m.rollout(bt["inputs"][1], bt["case_params"][1], bt["mask"][1], steps)
    assert one.shape == (steps, 1, 2) + tuple(bt["inputs"].shape[-2:])


def test_mask_requiring_grad_raises():
    sd, bt, gseq = _case(81, "cavity", 2, 5, 2)
    m = _model(sd, 5, 4, "float32")
    mask = bt["mask"].clone().requires_grad_(True)
    with pytest.raises(NotImplementedError):
        m.rollout(bt["inputs"], bt["case_params"], mask, 2)
    with pytest.raises(ValueError):
        m.rollout(bt["inputs"], bt["case_params"], bt["mask"], 0)


def _peak_bytes(fn):
    """Peak allocated bytes of fn() above what was allocated before it, with every model cache dropped first."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("where,act", [("cavity", "bfloat16"), ("tube", "float32")])
def test_memory_does_not_grow_with_steps_beyond_the_frames(where, act):
    """Peak memory of forward + backward at B = 64, K = 2 vs K = 8, from a cold model (workspaces, saved set and graph
    buffers included).  Per added step `rollout` holds frames only: its prediction, the loss's elementwise product and
    its gradient, and the captured graphs' static copies of the frame sequence (forward, backward) and of its gradient
    -- at most 6 frames.  Chained `generate` keeps one saved set per step."""
    b, depth = 64, 4
    sd, bt, _ = _case(91, where, b, 5, 8, depth)
    m = _model(sd, 5, depth, act)
    gh, gw = bt["inputs"].shape[-2:]
    frame = b * 2 * gh * gw * 4
    elt = 2 if act == "bfloat16" else 4
    saved_set = (depth + 1) * b * 32 * gh * gw * elt + depth * b * 32 * gh * gw * 4 + depth * 288 * b * 32 * 8

    def run(fn, steps):
        g = torch.randn(steps, b, 2, gh, gw, device="cuda")

        def body():
            x = bt["inputs"].clone().requires_grad_(True)
            (fn(x, steps) * g).sum().backward()
        m.invalidate_packed()
        m.zero_grad(set_to_none=True)
        return _peak_bytes(body)

    def roll(x, steps):
        return m.rollout(x, bt["case_params"], bt["mask"], steps)

    def chain(x, steps):
        preds = []
        for _ in range(steps):
            x = m.generate(x, bt["case_params"], bt["mask"])
            preds.append(x)
        return torch.stack(preds)

    d_roll = run(roll, 8) - run(roll, 2)
    d_chain = run(chain, 8) - run(chain, 2)
    _report(f"memory-{where}-{act}", {"frame_MB": frame / 1e6, "saved_set_MB": saved_set / 1e6,
                                       "rollout_K2_to_K8_MB": d_roll / 1e6, "chained_K2_to_K8_MB": d_chain / 1e6,
                                       "rollout_frames_per_step": d_roll / frame / 6})
    assert d_roll <= 6 * 6 * frame + (64 << 20), d_roll
    assert d_chain >= 6 * saved_set, d_chain


def test_fused_adam_on_a_four_step_rollout_loss_lowers_it():
    """Train a student through K = 4 rollouts towards a teacher's rollouts (seeded synthetic case)."""
    from cfdbench_b200 import FusedAdam
    steps, b, p = 4, 16, 5
    sd_t, bt, _ = _case(101, "cavity", b, p, steps)
    teacher = _model(sd_t, p, 4, "bfloat16")
    with torch.no_grad():
        target = teacher.rollout(bt["inputs"], bt["case_params"], bt["mask"], steps)
    student = _model(synth.make_state_dict(102, n_params=p, depth=4, spectral_gain=50.0), p, 4, "bfloat16")
    opt = FusedAdam(student.parameters(), lr=2e-3)
    losses = []
    for _ in range(30):
        seq = student.rollout(bt["inputs"], bt["case_params"], bt["mask"], steps)
        loss = ((seq - target) ** 2).mean() / (target ** 2).mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    _report("fused-adam-K4", {"first": losses[0], "last": losses[-1]})
    assert np.isfinite(losses).all() and losses[-1] < 0.5 * losses[0], losses


# ------------------------------------------------------------------------------- data parallel (2 GPUs)
def _dp_worker(rank, world, port, tmp):
    import torch.distributed as dist
    from cfdbench_b200 import dp
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    dp.init_from_env("nccl")
    torch.cuda.set_device(rank)
    p, steps, b = 5, 3, 8
    sd, bt, gseq = _case(111, "cavity", b, p, steps)
    lo, hi = dp.shard_range(b, rank, world)
    m = _model(sd, p, 4, "float32")
    m.enable_data_parallel()
    shard = {k: v[lo:hi] for k, v in bt.items()}
    _, got, _, _ = _rollout_grads(m, shard, gseq[:, lo:hi].contiguous(), steps)
    ref = None
    for r in range(world):
        a, c = dp.shard_range(b, r, world)
        m2 = _model(sd, p, 4, "float32")
        _, g, _, _ = _rollout_grads(m2, {k: v[a:c] for k, v in bt.items()}, gseq[:, a:c].contiguous(), steps)
        ref = g if ref is None else [x + y for x, y in zip(ref, g)]
    for (k, _), a, r in zip(m.named_parameters(), got, ref):
        e = (a - r / world).abs().max().item() / (r.abs().max().item() / world + 1e-30)
        assert e < 1e-5, (k, e)
    dist.barrier()
    dist.destroy_process_group()
    open(os.path.join(tmp, f"ok{rank}"), "w").write("ok")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_dp_rollout_gradients_are_the_mean_of_shard_gradients(tmp_path):
    import torch.multiprocessing as mp
    port = 29800 + os.getpid() % 1000
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert os.path.exists(tmp_path / "ok0") and os.path.exists(tmp_path / "ok1")
