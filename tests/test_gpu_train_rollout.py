"""`train_auto(rollout_steps=K)` -- training through K-step rollouts with every step replayed from a CUDA graph --
against the eager loop a user writes with `DeviceFrames.rollout_batch` + `Fno2d.rollout`: the window gather and the
fused K-step loss bit for bit against their single-step counterparts, bit identity of parameters, optimizer state and
losses after 3 epochs, no window across a case, the chain check, one synchronisation per epoch, memory, and a run that
lowers the 20-step rollout error."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from cfdbench_b200 import _lib, synth
from test_gpu_eval_auto import _model

pytestmark = pytest.mark.gpu


class _ChainSplit(torch.utils.data.Dataset):
    """A split laid out as the reference's auto datasets lay it out: per case T_c frames (u, v, mask),
    inputs = frames[:-s], labels = frames[s:], the cases one after another, and a `time_step_size` attribute.
    chain_across: the first frame of each case is the last frame of the previous one, so that the frames also chain
    across the case boundary and only the case ids tell a window that crosses it."""

    def __init__(self, lengths, problem="cavity", s=1, seed=0, chain_across=False):
        rng = np.random.default_rng(seed)
        gh, gw = synth.grid(problem)
        masks = synth.make_mask(rng, len(lengths), problem)[:, 0]
        ins, labs, ids = [], [], []
        last = None
        for c, t in enumerate(lengths):
            fr = np.empty((t, 3, gh, gw), np.float32)
            fr[:, :2] = np.clip(rng.standard_normal((t, 2, gh, gw)), -3, 3)
            if chain_across and last is not None:
                fr[0, :2] = last
            fr[:, 2] = masks[c]
            last = fr[-1, :2].copy()
            ins.append(fr[:-s])
            labs.append(fr[s:])
            ids += [c] * (t - s)
        self.inputs, self.labels = torch.from_numpy(np.concatenate(ins)), torch.from_numpy(np.concatenate(labs))
        self.case_ids = np.asarray(ids)
        self.time_step_size = s
        p = synth.n_case_params(problem)
        self.case_params = [dict(rotated=c % 2, **{f"p{j}": float(rng.standard_normal()) for j in range(p)}, dx=0.1)
                            for c in range(len(lengths))]

    def __len__(self):
        return len(self.inputs)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ window gather
@pytest.mark.parametrize("problem", ["cavity", "tube"])
@pytest.mark.parametrize("frame_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("b", [1, 7, 256])
def test_gather_window_matches_numpy_indexing(problem, frame_dtype, b):
    from cfdbench_b200 import DeviceFrames, rollout_windows
    lib = _lib.load()
    K, s = 3, 2
    ds = _ChainSplit([14, 9, 20], problem, s=s, seed=3)
    fr = DeviceFrames(ds, device="cuda", frame_dtype=frame_dtype)
    assert fr.time_step_size == s
    gh, gw, p = fr.height, fr.width, fr.n_case_params
    v = rollout_windows(ds.case_ids, K, s)
    idx = np.random.default_rng(b).choice(v, size=b, replace=True)
    fin = fr.frames_in.float().cpu().numpy()
    fout = fr.frames_out.float().cpu().numpy()
    mask = fin[idx, 2:3]
    ref_labels = np.stack([fout[idx + k * s, :2] * mask for k in range(K)])
    ref_cp = fr.case_table.cpu().numpy()[ds.case_ids[idx]]
    guard = 7
    sentinel = float.fromhex("-0x1.5p+99")

    def buf(*shape):
        return torch.full((int(np.prod(shape)) + 2 * guard,), sentinel, device="cuda")
    bi, bl, bm, bc, bs = buf(b, 2, gh, gw), buf(b, 2, gh, gw), buf(b, 1, gh, gw), buf(b, p), buf(K, b, 2, gh, gw)
    # keep the 64x64 path's outputs 16-byte aligned: offset every buffer by a multiple of 4 floats
    off = 8 if (gh, gw) == (64, 64) else guard
    view = {k: t[off:off + t.numel() - 2 * guard] for k, t in dict(i=bi, l=bl, m=bm, c=bc, s=bs).items()}
    idx_d = torch.as_tensor(idx, device="cuda")
    args = (fr.frames_in.data_ptr(), fr.frames_out.data_ptr(), fr.case_table.data_ptr(), fr.case_ids.data_ptr(),
            idx_d.data_ptr(), b, p, _lib.ACT_BF16 if frame_dtype == torch.bfloat16 else _lib.ACT_F32,
            view["i"].data_ptr(), view["l"].data_ptr(), view["m"].data_ptr(), view["c"].data_ptr(), K, s, fr.n,
            view["s"].data_ptr())
    if (gh, gw) == (64, 64):
        assert lib.fno_gather_window(*args, _st()) == 0
    else:
        assert lib.fno_grid_gather_window(*args, gh, gw, _st()) == 0
    torch.cuda.synchronize()
    got = {k: t.cpu().numpy() for k, t in view.items()}
    assert np.array_equal(got["i"].reshape(b, 2, gh, gw), fin[idx, :2])
    assert np.array_equal(got["m"].reshape(b, 1, gh, gw), mask)
    assert np.array_equal(got["l"].reshape(b, 2, gh, gw), fout[idx, :2])
    assert np.array_equal(got["c"].reshape(b, p), ref_cp)
    assert np.array_equal(got["s"].reshape(K, b, 2, gh, gw).view(np.uint32), ref_labels.view(np.uint32))
    for t in (bi, bl, bm, bc, bs):   # nothing written outside the outputs
        h = t.cpu().numpy()
        n_out = h.size - 2 * guard
        assert np.all(h[:off] == sentinel) and np.all(h[off + n_out:] == sentinel)
    # the same start samples through fno_gather_batch, and the Python wrapper
    ref = fr.batch(idx)
    rb = fr.rollout_batch(idx, K)
    for key in ("inputs", "label", "mask", "case_params"):
        assert torch.equal(rb[key], ref[key]), key
    assert torch.equal(rb["inputs"].flatten(), view["i"]) and torch.equal(rb["labels"].flatten(), view["s"])
    assert torch.equal(rb["labels"][0], ref["label"] * ref["mask"])


def test_gather_window_leaves_windows_past_the_split_untouched():
    from cfdbench_b200 import DeviceFrames
    lib = _lib.load()
    ds = _ChainSplit([12, 10], "tube", s=1, seed=4)
    fr = DeviceFrames(ds, device="cuda")
    gh, gw, p, K = fr.height, fr.width, fr.n_case_params, 4
    idx = torch.tensor([0, fr.n - 3, 5], device="cuda")   # the middle window needs sample n
    outs = [torch.full(shape, 1234.5, device="cuda") for shape in
            ((3, 2, gh, gw), (3, 2, gh, gw), (3, 1, gh, gw), (3, p), (K, 3, 2, gh, gw))]
    assert lib.fno_grid_gather_window(fr.frames_in.data_ptr(), fr.frames_out.data_ptr(), fr.case_table.data_ptr(),
                                      fr.case_ids.data_ptr(), idx.data_ptr(), 3, p, _lib.ACT_F32,
                                      *[t.data_ptr() for t in outs[:4]], K, 1, fr.n, outs[4].data_ptr(), gh, gw,
                                      _st()) == 0
    for t in outs[:4]:
        assert torch.all(t[1] == 1234.5) and not torch.any(t[0] == 1234.5)
    assert torch.all(outs[4][:, 1] == 1234.5) and not torch.any(outs[4][:, 0] == 1234.5)
    with pytest.raises(IndexError):
        fr.rollout_batch([fr.n - 3], K)


# ------------------------------------------------------------------------------------------------ fused K-step loss
@pytest.mark.parametrize("gh,gw,b", [(64, 64, 5), (66, 65, 3), (25, 127, 3), (25, 127, 1)])
@pytest.mark.parametrize("K", [1, 3, 4])
def test_loss_seq_matches_single_step_losses(gh, gw, b, K):
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(gh * K + b)
    preds = torch.randn(K, b, 2, gh, gw, device="cuda", generator=g)
    labels = torch.randn(K, b, 2, gh, gw, device="cuda", generator=g)
    labels[..., :3, :] = 0.0   # masked-out rows, as the targets have
    n = b * 2 * gh * gw
    scratch = torch.zeros(lib.fno_loss_seq_scratch_bytes(K), dtype=torch.uint8, device="cuda")
    out = torch.full((K + 1, 5), float("nan"), device="cuda")
    one = torch.zeros(lib.fno_loss_scratch_bytes(), dtype=torch.uint8, device="cuda")
    for rep in range(2):   # the scratch is left ready for the next call
        assert lib.fno_loss_seq_fwd(preds.data_ptr(), labels.data_ptr(), n, K, scratch.data_ptr(), out.data_ptr(),
                                    _st()) == 0
        rows = []
        for k in range(K):
            pk, lk = preds[k].clone(), labels[k].clone()   # aligned copies: fno_loss_fwd needs 16-byte alignment
            r = torch.empty(5, device="cuda")
            assert lib.fno_loss_fwd(pk.data_ptr(), lk.data_ptr(), n, one.data_ptr(), r.data_ptr(), _st()) == 0
            rows.append(r)
            assert torch.equal(out[k], r), (rep, k)
        agg = sum(r for r in rows) / K   # what the eager loop's sum(...) / K computes on the device
        assert torch.equal(out[K], agg), (out[K], agg)
    f64 = torch.stack(rows).double().mean(0)
    assert torch.allclose(out[K].double(), f64, rtol=1e-6, atol=0)
    # backward: dpreds_k = fno_loss_bwd(preds_k, labels_k, out_k, gout / K)
    gout = torch.randn(4, device="cuda", generator=g)
    dseq = torch.full_like(preds, float("nan"))
    assert lib.fno_loss_seq_bwd(preds.data_ptr(), labels.data_ptr(), out.data_ptr(), gout.data_ptr(), dseq.data_ptr(), n,
                                K, _st()) == 0
    gk = gout / K
    for k in range(K):
        pk, lk, dk = preds[k].clone(), labels[k].clone(), torch.empty_like(preds[k])
        assert lib.fno_loss_bwd(pk.data_ptr(), lk.data_ptr(), out[k].data_ptr(), gk.data_ptr(), dk.data_ptr(), n,
                                _st()) == 0
        assert torch.equal(dseq[k], dk), k


def test_loss_seq_backward_matches_autograd_of_the_mean():
    """gout * (1/K) is the gradient autograd hands each step's MseLoss for sum(nmse_k) / K."""
    from cfdbench_b200.loss import MseLoss
    lib = _lib.load()
    K, shape = 3, (2, 2, 64, 64)
    preds = torch.randn(K, *shape, device="cuda")
    labels = torch.randn(K, *shape, device="cuda")
    p = preds.clone().requires_grad_(True)
    loss_fn = MseLoss(normalize=True)
    ls = [loss_fn(preds=p[k], labels=labels[k]) for k in range(K)]
    (sum(l["nmse"] for l in ls) / K).backward()
    n = preds[0].numel()
    scratch = torch.zeros(lib.fno_loss_seq_scratch_bytes(K), dtype=torch.uint8, device="cuda")
    out, gout = torch.empty(K + 1, 5, device="cuda"), torch.tensor([0.0, 0.0, 0.0, 1.0], device="cuda")
    dseq = torch.empty_like(preds)
    assert lib.fno_loss_seq_fwd(preds.data_ptr(), labels.data_ptr(), n, K, scratch.data_ptr(), out.data_ptr(), _st()) == 0
    assert lib.fno_loss_seq_bwd(preds.data_ptr(), labels.data_ptr(), out.data_ptr(), gout.data_ptr(), dseq.data_ptr(), n, K,
                                _st()) == 0
    assert torch.equal(dseq, p.grad)
    assert torch.equal(out[K, 3], sum(l["nmse"] for l in ls).detach() / K)


# ------------------------------------------------------------------------------------------------ against the eager loop
def _eager_rollout_loop(model, frames, windows, K, num_epochs, lr, lr_step_size, lr_gamma, batch_size, eval_interval,
                        generator):
    """The loop a user writes with the drop-in pieces: window starts in DataLoader order, rollout_batch, model.rollout,
    sum(nmse_k) / K, backward, FusedAdam.step, zero_grad, .item(), a real StepLR and the evaluation loader's RNG draw."""
    from cfdbench_b200 import FusedAdam
    from cfdbench_b200.data import index_batches
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=lr_step_size, gamma=lr_gamma)
    losses = []
    for ep in range(num_epochs):
        for ib in index_batches(len(windows), batch_size, True, generator):
            b = frames.rollout_batch(windows[ib], K)
            preds = model.rollout(b["inputs"], b["case_params"], b["mask"], K)
            loss = sum(model.loss_fn(preds=preds[k], labels=b["labels"][k])["nmse"] for k in range(K)) / K
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss.item())
        sched.step()
        if (ep + 1) % eval_interval == 0:
            dev_eval_draw(generator)
    return losses, opt


CASES = [  # problem, act_dtype, case lengths, s, K, batch_size, lr_gamma, explicit generator
    ("cavity", "float32", (9, 14, 7), 1, 2, 8, 0.5, True),      # ragged last batch
    ("cavity", "bfloat16", (12, 10), 2, 4, 4, 0.9, False),
    ("cavity", "float32", (8, 9), 1, 4, 1, 0.9, True),          # B = 1
    ("cylinder", "float32", (10, 11), 1, 2, 8, 0.9, True),
    ("tube", "float32", (9, 8, 10), 1, 2, 8, 0.9, True),
    ("cavity", "float32", (6, 7), 1, 4, 16, 0.9, True),        # |V| < B: one ragged batch per epoch
]


@pytest.mark.parametrize("problem,act_dtype,lengths,s,K,batch_size,lr_gamma,explicit", CASES)
def test_train_auto_rollout_is_bit_identical_to_the_eager_loop(tmp_path, problem, act_dtype, lengths, s, K, batch_size,
                                                               lr_gamma, explicit):
    from cfdbench_b200 import DeviceFrames, rollout_windows, train_auto
    from test_gpu_eval_auto import _AutoSplit
    epochs, eval_interval = 3, 2
    ds, dev = _ChainSplit(lengths, problem, s=s, seed=21), _AutoSplit(4, problem, seed=22)
    windows = rollout_windows(ds.case_ids, K, s)
    ref_m, m = _model(problem, act_dtype, seed=8), _model(problem, act_dtype, seed=8)
    frames = DeviceFrames(ds, device="cuda")
    seed = 99
    kw = dict(num_epochs=epochs, lr=1e-3, lr_gamma=lr_gamma, batch_size=batch_size, eval_batch_size=3,
              eval_interval=eval_interval, rollout_steps=K)
    if explicit:
        ref_losses, ref_opt = _eager_rollout_loop(ref_m, frames, windows, K, epochs, 1e-3, 1, lr_gamma, batch_size,
                                                  eval_interval, torch.Generator().manual_seed(seed))
        out = train_auto(m, ds, dev, tmp_path, generator=torch.Generator().manual_seed(seed), **kw)
    else:
        torch.manual_seed(seed)
        ref_losses, ref_opt = _eager_rollout_loop(ref_m, frames, windows, K, epochs, 1e-3, 1, lr_gamma, batch_size,
                                                  eval_interval, None)
        torch.manual_seed(seed)
        out = train_auto(m, ds, dev, tmp_path, **kw)
    losses, opt = out["train_losses"], out["optimizer"]
    steps = -(-len(windows) // batch_size)
    assert len(losses) == len(ref_losses) == epochs * steps
    print(f"{problem} {act_dtype} K={K} |V|={len(windows)} B={batch_size}: max |loss diff| "
          f"{max(abs(a - b) for a, b in zip(losses, ref_losses)):.3e}")
    assert losses == ref_losses
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        sa, sb = opt.state[a], ref_opt.state[b]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]), name
        assert torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert torch.equal(sa["step"], sb["step"]) and float(sa["step"]) == epochs * steps
    assert opt.param_groups[0]["lr"] == ref_opt.param_groups[0]["lr"]


def test_train_auto_rollout_frozen_parameters_match_the_eager_loop(tmp_path):
    from cfdbench_b200 import DeviceFrames, rollout_windows, train_auto
    from test_gpu_eval_auto import _AutoSplit
    frozen = ("fc0.weight", "blocks.1.conv0.weights2", "blocks.2.w0.bias", "fc2.bias")
    ds, dev = _ChainSplit((10, 12), "cavity", seed=5), _AutoSplit(4, "cavity", seed=6)
    ref_m, m = _model("cavity", seed=4), _model("cavity", seed=4)
    for model in (ref_m, m):
        for name, prm in model.named_parameters():
            prm.requires_grad_(name not in frozen)
    init = {k: v.detach().clone() for k, v in m.named_parameters()}
    windows = rollout_windows(ds.case_ids, 3, 1)
    ref_losses, ref_opt = _eager_rollout_loop(ref_m, DeviceFrames(ds, device="cuda"), windows, 3, 3, 1e-3, 1, 0.9, 8,
                                              1000, torch.Generator().manual_seed(7))
    out = train_auto(m, ds, dev, tmp_path, num_epochs=3, batch_size=8, eval_interval=1000, rollout_steps=3,
                     generator=torch.Generator().manual_seed(7))
    assert out["train_losses"] == ref_losses
    opt = out["optimizer"]
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        if name in frozen:
            assert torch.equal(a, init[name]) and a not in opt.state, name
        else:
            assert not torch.equal(a, init[name]), name
            for k in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(opt.state[a][k], ref_opt.state[b][k]), (name, k)


def test_rollout_steps_1_is_the_single_step_loop(tmp_path):
    from cfdbench_b200 import train_auto
    from test_gpu_eval_auto import _AutoSplit
    ds, dev = _AutoSplit(21, "cavity", seed=1), _AutoSplit(4, "cavity", seed=2)
    outs, models = [], []
    for kw in ({}, dict(rollout_steps=1)):
        m = _model("cavity", seed=3)
        outs.append(train_auto(m, ds, dev, tmp_path / str(len(kw)), num_epochs=3, batch_size=8, eval_interval=2,
                               generator=torch.Generator().manual_seed(4), **kw))
        models.append(m)
    assert outs[0]["train_losses"] == outs[1]["train_losses"]
    for a, b in zip(models[0].parameters(), models[1].parameters()):
        assert torch.equal(a, b)


def test_windows_never_cross_a_case(tmp_path):
    """The frames chain across the case boundaries too, so the chain check would pass a crossing window; the case
    parameters differ, so one would change the loss.  train_auto visits rollout_windows' starts only."""
    from cfdbench_b200 import DeviceFrames, rollout_windows, train_auto
    from test_gpu_eval_auto import _AutoSplit
    ds = _ChainSplit((6, 5, 7), "cavity", seed=8, chain_across=True)
    K = 3
    windows = rollout_windows(ds.case_ids, K, 1)
    assert windows.tolist() == [0, 1, 2, 5, 6, 9, 10, 11, 12]   # the cases hold samples 0-4, 5-8 and 9-14
    frames = DeviceFrames(ds, device="cuda")
    with pytest.raises(ValueError, match="crosses a case boundary"):
        frames.rollout_batch([4], K)
    ref_m, m = _model("cavity", seed=2), _model("cavity", seed=2)
    ref_losses, _ = _eager_rollout_loop(ref_m, frames, windows, K, 2, 1e-3, 1, 0.9, 64, 1000,
                                        torch.Generator().manual_seed(1))
    out = train_auto(m, ds, _AutoSplit(3, "cavity", seed=1), tmp_path, num_epochs=2, batch_size=64, eval_interval=1000,
                     rollout_steps=K, generator=torch.Generator().manual_seed(1))
    assert out["train_losses"] == ref_losses and len(ref_losses) == 2
    for a, b in zip(m.parameters(), ref_m.parameters()):
        assert torch.equal(a, b)


def test_chain_check_refuses_permuted_samples(tmp_path):
    from cfdbench_b200 import train_auto
    from test_gpu_eval_auto import _AutoSplit
    ds = _ChainSplit((8, 10), "cavity", seed=9)
    ds.inputs[[11, 12]] = ds.inputs[[12, 11]].clone()
    ds.labels[[11, 12]] = ds.labels[[12, 11]].clone()
    m = _model("cavity", seed=1)
    init = [p.detach().clone() for p in m.parameters()]
    with pytest.raises(ValueError, match=r"does not chain .* sample 11's input frame is not sample 10's label frame"):
        train_auto(m, ds, _AutoSplit(3, "cavity"), tmp_path, num_epochs=1, batch_size=4, rollout_steps=2)
    assert all(torch.equal(a, b) for a, b in zip(m.parameters(), init))
    # single-step training does not need the chain
    train_auto(m, ds, _AutoSplit(3, "cavity"), tmp_path, num_epochs=1, batch_size=4, eval_interval=1000)


# ------------------------------------------------------------------------------------------------ syncs, memory
def _count_syncs(fn):
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(prev)
    return [str(w.message) for w in caught if "called a synchronizing CUDA operation" in str(w.message)]


def test_train_auto_rollout_syncs_and_memory(tmp_path):
    from cfdbench_b200 import DeviceFrames, train_auto
    from test_gpu_eval_auto import _AutoSplit
    m = _model("cavity", seed=6)
    dev = DeviceFrames(_AutoSplit(4, "cavity", seed=1), device="cuda")
    tr = DeviceFrames(_ChainSplit((20, 24, 22), "cavity", seed=2), device="cuda")

    def run(epochs, K):
        return train_auto(m, tr, dev, tmp_path, num_epochs=epochs, batch_size=8, eval_interval=1000, rollout_steps=K)
    run(1, 2)
    counts = {}
    for epochs in (1, 3):
        syncs = _count_syncs(lambda: run(epochs, 2))
        print(f"{epochs} epochs: {len(syncs)} synchronising operations", syncs[:3])
        counts[epochs] = len(syncs)
    assert counts == {1: 2, 3: 4}   # one per epoch plus the chain check

    def rise(epochs, K):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(epochs, K)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    r2, r6 = rise(2, 4), rise(6, 4)
    k2, k8 = rise(2, 2), rise(2, 8)
    frame = 2 * 64 * 64 * 4
    print(f"peak rise: 2 epochs {r2} B, 6 epochs {r6} B; K=2 {k2} B, K=8 {k8} B "
          f"({(k8 - k2) / (6 * 8 * frame):.2f} frames per sample per added step)")
    assert r6 <= r2 + 4096
    assert k8 - k2 <= 6 * 8 * 5 * frame


# ------------------------------------------------------------------------------------------------ it helps rollouts
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


def test_rollout_training_lowers_the_20_step_error(tmp_path):
    from cfdbench_b200 import infer_multistep, train_auto
    tr, test = _Dynamics(6, 24, seed=1), _Dynamics(3, 22, seed=2)
    nmse = {}
    for K in (1, 4):
        m = _model("cavity", seed=5)
        train_auto(m, tr, test, tmp_path / str(K), num_epochs=8, batch_size=8, eval_interval=1000, rollout_steps=K,
                   generator=torch.Generator().manual_seed(0))
        cps = [torch.tensor([0.1 * j for j in range(5)]) for _ in test.all_features]
        res = infer_multistep(m, test.all_features, cps, infer_steps=20)
        nmse[K] = [r["nmse"] for r in res]
        print(f"K={K}: 20-step nmse step 1 {nmse[K][0]:.4g}, step 20 {nmse[K][-1]:.4g}, mean {np.mean(nmse[K]):.4g}")
    assert np.all(np.isfinite(nmse[4])) and nmse[4][-1] < nmse[1][-1]
