"""Gradient-norm clipping and the EMA of the weights on the GPU: the norm kernel against float64 on real training
gradients, FusedAdam's clipping against clip_grad_norm_ + torch.optim.Adam, the EMA against a float64 recurrence with a
derived bound, train_auto's graphs against the eager loop bit for bit, and the EMA checkpoints."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from cfdbench_b200 import DeviceFrames, FusedAdam, RolloutNoise, _lib, add_input_noise, synth, train_auto
from test_gpu_eval_auto import _AutoSplit, _model
from test_gpu_train_rollout import _ChainSplit

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.path.join(ROOT, "oracle", "_ref", "src")
U32 = 2.0 ** -24   # float32 unit roundoff
U64 = 2.0 ** -53


def _real(t):
    return torch.view_as_real(t) if t.is_complex() else t


def _trained_grads(problem, act_dtype="float32", num_layers=4, b=8, frozen=()):
    """The parameters of a model after one real training backward (model(**batch), loss["nmse"].backward())."""
    from cfdbench_b200 import Fno2d
    from cfdbench_b200.loss import loss_name_to_fn
    p = synth.n_case_params(problem)
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=num_layers,
              hidden_dim=32, modes1=12, modes2=12, act_dtype=act_dtype)
    sd = synth.make_state_dict(3, n_params=p, depth=num_layers, spectral_gain=20.0)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m = m.cuda()
    for name, prm in m.named_parameters():
        prm.requires_grad_(name not in frozen)
    frames = DeviceFrames(_AutoSplit(b, problem, seed=4), device="cuda")
    m(**frames.batch(list(range(b))))["loss"]["nmse"].backward()
    return m


def _norm64(params):
    return float(np.sqrt(sum(float((_real(p.grad).double() ** 2).sum()) for p in params if p.grad is not None)))


def _torch_coef(norm, max_norm):
    """clip_grad_norm_'s coefficient from a float32 norm, as torch computes it on the device."""
    total = torch.tensor(norm, dtype=torch.float32, device="cuda")
    return float(torch.clamp(max_norm / (total + 1e-6), max=1.0))


def _launch_norm(params, max_norm, scratch):
    ps = [p for p in params if p.grad is not None]
    tables = FusedAdam._tables(ps, [p.grad for p in ps])
    arr = (_lib.FnoAdamTensors * len(tables))(*tables)
    out = torch.full((2,), -1.0, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.load().fno_grad_norm(arr, len(tables), max_norm, out.data_ptr(), scratch.data_ptr(), None, 0, None, st),
               "fno_grad_norm")
    return out.cpu(), len(tables)


# ------------------------------------------------------------------------------------------------ 1. the norm kernel
@pytest.mark.parametrize("problem,act_dtype,num_layers", [("cavity", "float32", 4), ("cavity", "bfloat16", 4),
                                                          ("tube", "float32", 4), ("cavity", "float32", 8)])
def test_grad_norm_against_float64(problem, act_dtype, num_layers):
    frozen = ("fc0.weight", "blocks.1.conv0.weights2") if num_layers == 4 else ()
    m = _trained_grads(problem, act_dtype, num_layers, frozen=frozen)
    params = list(m.parameters())
    scratch = torch.zeros(_lib.load().fno_grad_norm_scratch_bytes() // 8 + 1, dtype=torch.float64, device="cuda")
    ref = _norm64(params)   # frozen parameters have no .grad: not counted
    n_terms = sum(_real(p.grad).numel() for p in params if p.grad is not None)
    for max_norm in (ref / 3, ref * 3):
        out, n_tables = _launch_norm(params, max_norm, scratch)
        norm, coef = float(out[0]), float(out[1])
        # float64 accumulation (n terms, relative n * u64) then the float32 rounding of the square root
        bound = ref * (U32 + n_terms * U64)
        print(f"{problem} {act_dtype} depth {num_layers}: {n_tables} tables, {n_terms} floats, norm {norm!r} vs float64 "
              f"{ref!r}: |err| {abs(norm - ref):.3e}, bound {bound:.3e}")
        assert abs(norm - ref) <= bound
        assert coef == _torch_coef(norm, max_norm)
        assert (coef == 1.0) == (max_norm > ref)
        again, _ = _launch_norm(params, max_norm, scratch)
        assert torch.equal(again, out)   # bit-reproducible (and the scratch was left re-armed)
    assert n_tables == (2 if num_layers == 8 else 1)
    if frozen:
        for name in frozen:
            assert dict(m.named_parameters())[name].grad is None
    # FusedAdam's clipping runs the same kernel over the same gradients
    opt = FusedAdam(m.parameters(), max_grad_norm=ref / 2)
    opt.step()
    assert float(opt.last_grad_norm) == norm


def test_grad_norm_non_finite_is_torchs():
    """error_if_nonfinite=False: an infinite norm gives coefficient 0, a NaN norm a NaN coefficient, as in torch."""
    scratch = torch.zeros(_lib.load().fno_grad_norm_scratch_bytes() // 8 + 1, dtype=torch.float64, device="cuda")
    for bad in (float("inf"), float("nan")):
        p = torch.nn.Parameter(torch.zeros(1000, device="cuda"))
        p.grad = torch.ones(1000, device="cuda")
        p.grad[17] = bad
        out, _ = _launch_norm([p], 1.0, scratch)
        total = torch.nn.utils.clip_grad_norm_([p], 1.0, error_if_nonfinite=False)
        for got, want in ((float(out[0]), float(total)), (float(out[1]), _torch_coef(float(total), 1.0))):
            assert got == want or (np.isnan(got) and np.isnan(want)), (bad, got, want)


# ------------------------------------------------------------------------------------------------ 2. clipping vs torch
def _params(seed):
    g = torch.Generator().manual_seed(seed)
    shapes = [(32, 10, 1, 1), (32,), (32, 32, 12, 12), (128, 32, 1, 1), (5,)]
    out = []
    for i, s in enumerate(shapes):
        t = torch.randn(s, generator=g) * 0.1
        if i == 2:
            t = torch.complex(t, torch.randn(s, generator=g) * 0.1)
        out.append(torch.nn.Parameter(t.cuda()))
    return out


@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_clipping_matches_clip_grad_norm_and_torch_adam(wd):
    pa, pb, pc = _params(1), _params(1), _params(1)
    max_norm = 1.0
    oa = FusedAdam(pa, lr=1e-3, weight_decay=wd, max_grad_norm=max_norm)
    ob = torch.optim.Adam(pb, lr=1e-3, weight_decay=wd)
    oc = FusedAdam(pc, lr=1e-3, weight_decay=wd)   # clipped by hand with our own coefficient: the clip is exact
    g = torch.Generator().manual_seed(9)
    bound = []
    b1, b2 = 0.9, 0.999
    # FusedAdam forms 1 - beta in float32 (torch in double): the moments differ from torch's by these relative amounts
    # with or without clipping
    d1 = abs(float(1 - np.float32(b1)) - (1 - b1)) / (1 - b1)
    d2 = abs(float(1 - np.float32(b2)) - (1 - b2)) / (1 - b2)
    M = [torch.zeros(_real(a).shape, dtype=torch.float64) for a in pa]   # sum of |terms| of exp_avg
    W = [torch.zeros(_real(a).shape, dtype=torch.float64) for a in pa]   # the same with the terms squared (exp_avg_sq)
    P = [torch.zeros(_real(a).shape, dtype=torch.float64) for a in pa]   # bound of |p_ours - p_torch|
    Mp = [torch.zeros_like(x) for x in P]   # what the weight decay of P adds to the moments' bounds
    Vp = [torch.zeros_like(x) for x in P]
    for step, scale in enumerate((3.0, 0.2, 10.0, 0.05, 1.5, 0.5)):   # the clip binds on steps 0, 2, 4
        grads = []
        for a in pa:
            gr = torch.randn(_real(a).shape, generator=g)
            grads.append(gr)
        raw = float(np.sqrt(sum(float((x.double() ** 2).sum()) for x in grads)))
        for a, b, c, gr in zip(pa, pb, pc, grads):
            gr = (gr * (scale / raw)).cuda()
            gr = torch.view_as_complex(gr) if a.is_complex() else gr
            a.grad, b.grad, c.grad = gr.clone(), gr.clone(), gr.clone()
        oa.step()
        norm = float(oa.last_grad_norm)
        total = torch.nn.utils.clip_grad_norm_(pb, max_norm)
        ob.step()
        coef = _torch_coef(norm, max_norm)
        if coef < 1:
            for c in pc:
                c.grad.mul_(coef)
        oc.step()
        binds = scale > max_norm
        assert (coef < 1) == binds and (float(total) > max_norm) == binds
        # the two norms differ by their summation order: torch's per-tensor float32 norms against one float64 sum
        rel = abs(norm - float(total)) / float(total)
        bound.append(rel)
        assert rel <= 8 * U32 * len(pa), (step, norm, float(total))
        tol = 4 * max(bound) + 16 * U32 * (step + 1)
        t = step + 1
        s_t, k_t = 1e-3 / (1 - b1 ** t), 1 / np.sqrt(1 - b2 ** t)   # Adam's step size and 1 / sqrt(bc2)
        for a, b, c, Mi, Wi, Pi, Mpi, Vpi in zip(pa, pb, pc, M, W, P, Mp, Vp):
            gi = _real(c.grad).double().cpu().abs() + wd * _real(c).double().cpu().abs()
            Mi.mul_(b1).add_((1 - b1) * gi)
            Wi.mul_(b2).add_((1 - b2) * gi ** 2)
            Mpi.mul_(b1).add_((1 - b1) * wd * Pi)
            Vpi.mul_(b2).add_((1 - b2) * 2 * (gi + wd * Pi) * wd * Pi)
            sa, sb, sc = oa.state[a], ob.state[b], oc.state[c]
            # our clip == multiplying the gradients by our coefficient first: bit for bit
            assert torch.equal(a, c) and torch.equal(sa["exp_avg"], sc["exp_avg"])
            assert torch.equal(sa["exp_avg_sq"], sc["exp_avg_sq"])
            # against torch: the clipped gradient g c + wd p differs by at most tol (g c + wd p), so exp_avg by tol
            # times the sum of its terms' moduli and exp_avg_sq by 2 tol times that of their squares (the weight decay
            # can cancel g c, so neither is relative to the moment itself).  A missing clip would put them off by the
            # factor scale / max_norm >= 1.5; the coefficients differ by the norms' relative difference above
            m_a, m_b = _real(sa["exp_avg"]).double().cpu(), _real(sb["exp_avg"]).double().cpu()
            v_a, v_b = _real(sa["exp_avg_sq"]).double().cpu(), _real(sb["exp_avg_sq"]).double().cpu()
            em = (tol + 2 * d1) * Mi + Mpi + 1e-30
            ev = 2 * tol * (1 + tol) * Wi + 2 * d2 * v_b + Vpi + 1e-30
            assert bool(((m_a - m_b).abs() <= em).all()), (step, "exp_avg")
            assert bool(((v_a - v_b).abs() <= ev).all()), (step, "exp_avg_sq")
            # the parameters: |m_a / D_a - m_b / D_b| <= em / D + (|m_b| + em) |D_a - D_b| / D^2 with D = sqrt(v) k + eps
            # at its smallest over the v interval, |sqrt(v_a) - sqrt(v_b)| <= min(ev / (2 sqrt(v_lo)), sqrt(ev)), plus
            # a few float32 roundings of the update.  Where the weight decay cancels g c the update is as sensitive as
            # Adam makes it, so this is not a relative bound
            v_lo = (v_b - ev).clamp(min=0)
            dsq = torch.minimum(ev / (2 * v_lo.sqrt()).clamp(min=1e-300), ev.sqrt())
            d_lo = v_lo.sqrt() * k_t + 1e-8
            u_hi = s_t * (m_b.abs() + em) / d_lo
            Pi.add_(s_t * (em / d_lo + (m_b.abs() + em) * k_t * dsq / d_lo ** 2) + 8 * U32 * u_hi)
            err_p = (_real(a).detach().double().cpu() - _real(b).detach().double().cpu()).abs()
            assert bool((err_p <= Pi + 2 * t * U32 * _real(b).detach().double().cpu().abs()).all()), (step, "param")
    print("norm relative differences against clip_grad_norm_:", [f"{r:.1e}" for r in bound])


def test_non_binding_clip_is_bit_identical_to_no_clip():
    pa, pb = _params(2), _params(2)
    oa, ob = FusedAdam(pa, lr=1e-3, max_grad_norm=1e6), FusedAdam(pb, lr=1e-3)
    g = torch.Generator().manual_seed(3)
    for _ in range(4):
        for a, b in zip(pa, pb):
            gr = torch.randn(_real(a).shape, generator=g).cuda()
            gr = torch.view_as_complex(gr) if a.is_complex() else gr
            a.grad, b.grad = gr.clone(), gr.clone()
        oa.step()
        ob.step()
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(oa.state[a][k], ob.state[b][k])


def _seeded_adam_inputs(seed):
    """_params(seed) with seeded gradients, exp_avg and exp_avg_sq (>= 0), and an independent copy of all of them."""
    g = torch.Generator().manual_seed(seed)
    ps, states = _params(seed), []
    for p in ps:
        def draw(scale, square=False):
            x = torch.randn(_real(p).shape, generator=g) * scale
            x = x * x if square else x
            return (torch.view_as_complex(x) if p.is_complex() else x).cuda()
        p.grad = draw(1.0)
        states.append(dict(exp_avg=draw(0.1), exp_avg_sq=draw(0.1, square=True)))
    qs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    for q, p in zip(qs, ps):
        q.grad = p.grad.clone()
    return (ps, states), (qs, [{k: v.clone() for k, v in st.items()} for st in states])


def _assert_same_bits(a, b):
    (pa, sa), (pb, sb) = a, b
    bits = lambda t: _real(t.detach()).contiguous().view(torch.int32)
    for x, y, u, v in zip(pa, pb, sa, sb):
        assert torch.equal(bits(x), bits(y))
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(bits(u[k]), bits(v[k])), k


def test_plain_adam_entry_points_match_their_ex_forms():
    """fno_adam_step is fno_adam_step_ex(..., NULL, NULL, 0.0) and fno_adam_step_dev is fno_adam_step_dev_ex(..., NULL,
    NULL, NULL), bit for bit; FusedAdam.step (which issues the _ex form) is direct fno_adam_step calls."""
    lib = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    lr, b1, b2, eps, wd = 1e-3, 0.9, 0.999, 1e-8, 0.01

    def tables(ps, states):
        return FusedAdam._tables(ps, [p.grad for p in ps], states)

    a, b = _seeded_adam_inputs(21)
    before = a[0][0].detach().clone()
    for step in (1, 2, 9):
        for t, u in zip(tables(*a), tables(*b)):
            assert lib.fno_adam_step(C.byref(t), lr, b1, b2, eps, wd, step, st) == 0
            assert lib.fno_adam_step_ex(C.byref(u), lr, b1, b2, eps, wd, step, None, None, 0.0, st) == 0
    _assert_same_bits(a, b)
    assert not torch.equal(a[0][0], before)

    a, b = _seeded_adam_inputs(22)
    n = 3
    coef = np.empty((n, 2), np.float32)
    assert lib.fno_adam_coefficients(lr, b1, b2, 4, n, coef.ctypes.data) == 0
    coef = torch.from_numpy(coef).cuda()
    cursor = torch.zeros(1, dtype=torch.int32, device="cuda")
    for c in range(n + 1):   # the last cursor is outside the table: both write nothing
        cursor.fill_(c)
        for t, u in zip(tables(*a), tables(*b)):
            assert lib.fno_adam_step_dev(C.byref(t), coef.data_ptr(), n, cursor.data_ptr(), b1, b2, eps, wd, st) == 0
            assert lib.fno_adam_step_dev_ex(C.byref(u), coef.data_ptr(), n, cursor.data_ptr(), b1, b2, eps, wd, None, None,
                                            None, st) == 0
    _assert_same_bits(a, b)

    a, b = _seeded_adam_inputs(23)
    opt = FusedAdam(a[0], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    for p, s in zip(*a):
        opt.state[p].update(step=torch.tensor(6.0), **s)
    for step in (7, 8):
        opt.step()
        for t in tables(*b):
            assert lib.fno_adam_step(C.byref(t), lr, b1, b2, eps, wd, step, st) == 0
    _assert_same_bits(a, b)
    assert all(float(opt.state[p]["step"]) == 8 for p in a[0])


# ------------------------------------------------------------------------------------------------ 3. EMA
@pytest.mark.parametrize("decay,steps", [(0.9, 40), (0.999, 25)])
def test_ema_against_a_float64_recurrence(decay, steps):
    """e_t = fmaf(-d, fl(p - e), p): the subtraction and the fma round once each, so with E the exact recurrence
    E_t = d E_{t-1} + (1 - d) p_t fed the same float32 p_t, |e_t - E_t| <= d |e_{t-1} - E_{t-1}| + u d |p_t - e_{t-1}|
    + u |e_t| (1 + 2u): the carried error is scaled by d_t and each step adds at most two roundings."""
    ps = _params(4)
    opt = FusedAdam(ps, lr=1e-2, ema_decay=decay)
    table = np.empty(steps, np.float32)
    assert _lib.load().fno_ema_decays(decay, 1, steps, table.ctypes.data) == 0
    g = torch.Generator().manual_seed(6)
    E = err_bound = prev = None
    worst = 0.0
    for t in range(1, steps + 1):
        for a in ps:
            gr = torch.randn(_real(a).shape, generator=g).cuda()
            a.grad = torch.view_as_complex(gr) if a.is_complex() else gr
        opt.step()
        p = [_real(a).detach().double().cpu() for a in ps]
        e = [_real(opt.state[a]["ema"]).double().cpu() for a in ps]
        d = float(table[t - 1])
        if t == 1:
            assert d == 0.0
            for a in ps:
                assert torch.equal(opt.state[a]["ema"], a)   # exactly the weights after the first step
            E, err_bound = p, [torch.zeros_like(x) for x in p]
        else:
            E = [d * Ek + (1 - d) * pk for Ek, pk in zip(E, p)]
            err_bound = [d * bk + U32 * d * (pk - ek0).abs() + U32 * ek.abs() * (1 + 2 * U32)
                         for bk, pk, ek0, ek in zip(err_bound, p, prev, e)]
        for ek, Ek, bk in zip(e, E, err_bound):
            err = (ek - Ek).abs()
            slack = 4 * U64 * (Ek.abs() + 1e-30)   # the float64 recurrence's own rounding
            assert bool((err <= bk * (1 + 1e-9) + slack).all()), (t, float((err - bk).max()))
            worst = max(worst, float((err / (bk + slack)).max()))
        prev = e
    assert float(table[-1]) <= decay and (decay > 0.99 or float(table[-1]) == np.float32(decay))
    print(f"decay {decay}: largest |err| / bound over {steps} steps {worst:.3f}")


# ------------------------------------------------------------------------------------------------ 4. graph == eager
def _eager_loop(model, frames, windows, K, G, sigma, noise_seed, every, num_epochs, lr, lr_gamma, batch_size,
                eval_interval, generator, **opts):
    """The loops of train_auto's docstring with FusedAdam(max_grad_norm=..., ema_decay=...)."""
    from cfdbench_b200.data import index_batches
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr, **opts)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=lr_gamma)
    losses, norms, t = [], [], 0
    for ep in range(num_epochs):
        for ib in index_batches(len(windows), batch_size, True, generator):
            t += 1
            noise = dict(noise_std=sigma, noise_seed=noise_seed, noise_step=t)
            if K == 1:
                loss = model(**frames.batch(windows[ib], **noise))["loss"]["nmse"]
            else:
                b = frames.rollout_batch(windows[ib], K, **noise)
                ids = torch.as_tensor(windows[ib], device="cuda")
                x = b["inputs"]
                rn = None
                if every:
                    for k in range(K - G):
                        if k > 0:
                            x = add_input_noise(x, b["mask"], ids, sigma, noise_seed, t, stream=k)
                        with torch.no_grad():
                            x = model.generate_many(x, b["case_params"], b["mask"], 1)[0]
                    rn = RolloutNoise(sigma, noise_seed, t, ids, K - G)
                elif K > G:
                    with torch.no_grad():
                        x = model.generate_many(x, b["case_params"], b["mask"], K - G)[-1]
                seq = model.rollout(x, b["case_params"], b["mask"], G, noise=rn)
                loss = sum(model.loss_fn(preds=seq[g], labels=b["labels"][K - G + g])["nmse"] for g in range(G)) / G
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


MODES = {"single": (1, 1, 0.0, False), "rollout": (3, 3, 0.0, False), "pushforward-noise": (3, 1, 0.05, True)}
GRIDS = {"cavity": ("cavity", "float32"), "cavity-bf16": ("cavity", "bfloat16"), "tube": ("tube", "float32")}


@pytest.mark.parametrize("opts", [dict(max_grad_norm=0.02, ema_decay=0.99)])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("grid", list(GRIDS))
def test_train_auto_is_bit_identical_to_the_eager_loop(tmp_path, grid, mode, opts):
    _graph_vs_eager(tmp_path, grid, mode, opts)


@pytest.mark.parametrize("opts", [dict(max_grad_norm=0.01), dict(ema_decay=0.9)])
def test_train_auto_one_option_is_bit_identical_to_the_eager_loop(tmp_path, opts):
    _graph_vs_eager(tmp_path, "cavity", "rollout", opts, frozen=("fc0.weight", "blocks.1.conv0.weights2", "fc2.bias"))


def _graph_vs_eager(tmp_path, grid, mode, opts, frozen=()):
    from cfdbench_b200 import rollout_windows
    problem, act_dtype = GRIDS[grid]
    K, G, sigma, every = MODES[mode]
    epochs, eval_interval, noise_seed, lr_gamma, batch_size = 3, 2, 77, 0.9, 8
    ds, dev = _ChainSplit((9, 12, 7), problem, s=1, seed=31), _AutoSplit(4, problem, seed=32)
    windows = rollout_windows(ds.case_ids, K, 1)
    ref_m, m = _model(problem, act_dtype, seed=8), _model(problem, act_dtype, seed=8)
    for model in (ref_m, m):
        for name, prm in model.named_parameters():
            prm.requires_grad_(name not in frozen)
    ref_losses, ref_norms, ref_opt = _eager_loop(ref_m, DeviceFrames(ds, device="cuda"), windows, K, G, sigma, noise_seed,
                                                 every, epochs, 1e-3, lr_gamma, batch_size, eval_interval,
                                                 torch.Generator().manual_seed(5), **opts)
    out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, lr_gamma=lr_gamma, batch_size=batch_size,
                     eval_batch_size=3, eval_interval=eval_interval, rollout_steps=K, rollout_grad_steps=G,
                     input_noise_std=sigma, noise_seed=noise_seed, noise_every_step=every,
                     generator=torch.Generator().manual_seed(5), **opts)
    losses, opt = out["train_losses"], out["optimizer"]
    assert losses == ref_losses
    clip = opts.get("max_grad_norm")
    if clip is not None:
        bound = sum(n > clip for n in ref_norms)
        print(f"{grid} {mode}: the clip bound on {bound} of {len(ref_norms)} steps, norms {min(ref_norms):.3g} .. "
              f"{max(ref_norms):.3g}")
        assert bound > 0
        assert out["grad_norms"] == ref_norms and len(ref_norms) == len(losses)
        assert json.load(open(tmp_path / "grad_norms.json")) == ref_norms
        assert float(opt.last_grad_norm) == ref_norms[-1]
    else:
        assert "grad_norms" not in out and not (tmp_path / "grad_norms.json").exists()
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        if name in frozen:
            assert a not in opt.state, name
            continue
        sa, sb = opt.state[a], ref_opt.state[b]
        for k in ("exp_avg", "exp_avg_sq", "step") + (("ema",) if "ema_decay" in opts else ()):
            assert torch.equal(sa[k], sb[k]), (name, k)
    if "ema_decay" in opts:
        for (name, e), a in zip(out["ema_model"].named_parameters(), m.parameters()):
            st = opt.state.get(a)
            assert torch.equal(e, st["ema"] if st else a), name
    else:
        assert "ema_model" not in out


# ------------------------------------------------------------------------------------------------ 5. checkpoints
def _get_best_ckpt(output_dir):
    best, best_dir = float("inf"), None
    for d in sorted(output_dir.glob("ckpt-*")):
        loss = json.load(open(d / "scores.json"))["dev_loss"]
        if loss < best:
            best, best_dir = loss, d
    return best_dir


_LOAD_BEST = r"""
import sys
sys.path.insert(0, {root!r})
sys.path.insert(0, {tests!r})
from cfdbench_b200 import runner
runner.install({src!r}, stub_missing=True)
from pathlib import Path
import torch
from utils.common import load_best_ckpt
from test_gpu_eval_auto import _model
m = _model("cavity", seed=1)
load_best_ckpt(m, Path({out!r}))
torch.save(m.state_dict(), {dst!r})
"""


@pytest.mark.parametrize("dev_rollout", [None, 3])
def test_ema_checkpoints(tmp_path, dev_rollout):
    from cfdbench_b200 import evaluate_auto, evaluate_rollout_auto
    tr, dv = _ChainSplit((14, 12, 15), "cavity", s=1, seed=21), _ChainSplit((12, 10), "cavity", s=1, seed=22)
    m = _model("cavity", seed=9)
    out_dir = tmp_path / "run"
    res = train_auto(m, tr, dv, out_dir, num_epochs=4, lr=2e-3, batch_size=8, eval_interval=2, log_interval=1000,
                     rollout_steps=2, ema_decay=0.95, max_grad_norm=0.5, dev_rollout_steps=dev_rollout,
                     generator=torch.Generator().manual_seed(3))
    ema_model, opt = res["ema_model"], res["optimizer"]
    assert ema_model is not m and ema_model.act_dtype == m.act_dtype and ema_model.device == m.device
    for a, e in zip(m.parameters(), ema_model.parameters()):
        assert torch.equal(e, opt.state[a]["ema"])
    assert any(not torch.equal(a, e) for a, e in zip(m.parameters(), ema_model.parameters()))   # model: trained weights
    losses = {}
    for c in ("ckpt-1", "ckpt-3"):
        fresh = _model("cavity", seed=1)
        fresh.load_state_dict(torch.load(out_dir / c / "model.pt", map_location="cpu"))
        sc = json.load(open(out_dir / c / "scores.json"))
        single = float(np.mean(evaluate_auto(fresh, DeviceFrames(dv, device="cuda"), batch_size=2)["scores"]["all"]["nmse"]))
        if dev_rollout is None:
            assert sc["dev_loss"] == single
        else:
            again = evaluate_rollout_auto(fresh, dv, dev_rollout)
            assert sc["dev_loss"] == again["loss"] and sc["dev_loss_single_step"] == single
        losses[c] = sc["dev_loss"]
    # the last checkpoint holds the final EMA weights
    last = torch.load(out_dir / "ckpt-3" / "model.pt", map_location="cpu")
    for k, v in ema_model.state_dict().items():
        assert torch.equal(last[k], v.cpu()), k
    assert _get_best_ckpt(out_dir).name == min(losses, key=losses.get)
    if os.path.isdir(os.path.join(REF_SRC, "utils")):   # the reference's own load_best_ckpt (installed by build())
        import shutil
        src = str(tmp_path / "src")
        shutil.copytree(REF_SRC, src)
        for root, dirs, files in os.walk(src):
            os.chmod(root, 0o755)
            for f in files:
                os.chmod(os.path.join(root, f), 0o644)
        dst = str(tmp_path / "best.pt")
        env = {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
               "PYTHONDONTWRITEBYTECODE": "1"}
        r = subprocess.run([sys.executable, "-c", _LOAD_BEST.format(root=ROOT, tests=os.path.join(ROOT, "tests"), src=src,
                                                                    out=str(out_dir), dst=dst)],
                           capture_output=True, text=True, env=env, cwd=src, timeout=600)
        assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
        got = torch.load(dst, map_location="cpu")
        best = torch.load(_get_best_ckpt(out_dir) / "model.pt", map_location="cpu")
        for k in best:
            assert torch.equal(got[k].cpu(), best[k]), k


def test_defaults_launch_what_they_launched(tmp_path):
    """With both options None the step graph issues the parent's launches: no norm and no _ex Adam kernel."""
    from torch.profiler import ProfilerActivity, profile
    tr, dv = _AutoSplit(16, "cavity", seed=1), _AutoSplit(4, "cavity", seed=2)
    names = {}
    for key, kw in (("none", {}), ("both", dict(max_grad_norm=1.0, ema_decay=0.9))):
        m = _model("cavity", seed=3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            train_auto(m, tr, dv, tmp_path / key, num_epochs=1, batch_size=8, eval_interval=1000, **kw)
            torch.cuda.synchronize()
        names[key] = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    print({k: sorted(n for n in v if "adam" in n or "norm" in n) for k, v in names.items()})
    assert not any("grad_norm_kernel" in n or "adam_step_ex_kernel" in n for n in names["none"])
    assert any("adam_step_kernel" in n for n in names["none"])
    assert any("grad_norm_kernel" in n for n in names["both"]) and any("adam_step_ex_kernel" in n for n in names["both"])
