"""Fno2d is differentiable w.r.t. its input frame and case parameters (fno_backward_inputs, lift_bwd_data_kernel), as
the reference is under plain autograd: single training steps, a frozen model (sensitivities / inverse problems), and
unrolled training through chained `generate` calls, against autograd of the CPU torch port of the reference."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(sd, p, act):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m


def _rel(a: torch.Tensor, ref: torch.Tensor) -> float:
    a, ref = a.detach().cpu().double(), ref.detach().cpu().double()
    return float((a - ref).norm() / ref.norm())


def _tol(act):
    # fp32 storage: the gradient contract of the parameter gradients (DESIGN.md 5); bf16 storage: against the port with
    # straight-through bf16 rounding, whose saved-activation noise is ~2^-9 * sqrt(depth)
    return 5e-5 if act == "float32" else 2e-2


def _round_fn(act):
    from oracle import fno_torch_port as port
    return None if act == "float32" else port.bf16_round_ste


def _step(m, tb, inputs_grad: bool):
    """One nmse.backward() through the module; returns (preds, d_inputs, d_case_params, parameter grads)."""
    x = tb["inputs"].clone().requires_grad_(inputs_grad)
    cp = tb["case_params"].clone().requires_grad_(inputs_grad)
    m.zero_grad(set_to_none=True)
    out = m(inputs=x, case_params=cp, mask=tb["mask"], label=tb["label"])
    out["loss"]["nmse"].backward()
    grads = {k: (None if v.grad is None else v.grad.detach().clone()) for k, v in m.named_parameters()}
    return out["preds"], x.grad, cp.grad, grads


@pytest.mark.parametrize("act", ["float32", "bfloat16"])
@pytest.mark.parametrize("problem", ["cavity", "cylinder"])
def test_single_step_and_frozen_model_input_gradients(problem, act):
    from cfdbench_b200 import synth
    from oracle import fno_torch_port as port
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(71, n_params=p, spectral_gain=50.0)
    batch = synth.make_batch(72, 6, problem)
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    m = _model(sd, p, act)

    _, _, _, g_params_only = _step(m, tb, inputs_grad=False)
    _, d_in, d_cp, g_all = _step(m, tb, inputs_grad=True)
    # the same step again: fixed-order reductions, no atomics -> bit-identical
    _, d_in2, d_cp2, _ = _step(m, tb, inputs_grad=True)
    assert torch.equal(d_in, d_in2) and torch.equal(d_cp, d_cp2)
    for k in g_params_only:   # asking for input gradients does not change the parameter gradients by a bit
        assert torch.equal(g_params_only[k], g_all[k]), k

    # the port of the reference, plain autograd
    pp = port.params_from_numpy(sd, requires_grad=True)
    cb = {k: torch.from_numpy(v) for k, v in batch.items()}
    xr = cb["inputs"].clone().requires_grad_(True)
    cr = cb["case_params"].clone().requires_grad_(True)
    o = port.forward(pp, xr, cr, cb["mask"], label=cb["label"], round_fn=_round_fn(act))
    o["loss"]["nmse"].backward()
    tol = _tol(act)
    assert d_in.shape == xr.shape and d_cp.shape == cr.shape
    assert _rel(d_in, xr.grad) < tol, _rel(d_in, xr.grad)
    assert _rel(d_cp, cr.grad) < tol, _rel(d_cp, cr.grad)
    for k, v in g_all.items():
        assert _rel(v, pp[k].grad) < tol, (k, _rel(v, pp[k].grad))

    # frozen model: the data-only backward gives the same input gradients, bit for bit, and no parameter gradient
    for prm in m.parameters():
        prm.requires_grad_(False)
    preds_f, d_in_f, d_cp_f, g_f = _step(m, tb, inputs_grad=True)
    assert preds_f.requires_grad and preds_f.grad_fn is not None
    assert torch.equal(d_in_f, d_in) and torch.equal(d_cp_f, d_cp)
    assert all(v is None for v in g_f.values())
    # only one of the two inputs asks
    x = tb["inputs"].clone().requires_grad_(True)
    m(inputs=x, case_params=tb["case_params"], mask=tb["mask"], label=tb["label"])["loss"]["nmse"].backward()
    assert torch.equal(x.grad, d_in)
    cp = tb["case_params"].clone().requires_grad_(True)
    m(inputs=tb["inputs"], case_params=cp, mask=tb["mask"], label=tb["label"])["loss"]["nmse"].backward()
    assert torch.equal(cp.grad, d_cp)


@pytest.mark.parametrize("act", ["float32", "bfloat16"])
def test_unrolled_rollout_training_matches_port(act):
    """x1 = generate(x0), x2 = generate(x1), x3 = generate(x2), loss summed over the steps: forward k+1 runs before
    backward k (each call keeps its own saved activations; the workspace scratch is shared in stream order).  B = 70
    gives the 32-sample project chunks of the backward a ragged tail."""
    from cfdbench_b200 import synth
    from oracle import fno_torch_port as port
    p, steps = 5, 3
    sd = synth.make_state_dict(81, n_params=p, spectral_gain=50.0)
    batch = synth.make_batch(82, 70, "cavity")
    rng = np.random.default_rng(83)
    weights = [torch.from_numpy(rng.standard_normal(batch["inputs"].shape).astype(np.float32)) for _ in range(steps)]
    m = _model(sd, p, act)
    x0 = torch.from_numpy(batch["inputs"]).cuda().requires_grad_(True)
    cp = torch.from_numpy(batch["case_params"]).cuda().requires_grad_(True)
    mask = torch.from_numpy(batch["mask"]).cuda()
    cur, loss = x0, 0.0
    for s in range(steps):
        cur = m.generate(cur, cp, mask)
        loss = loss + (cur * weights[s].cuda()).sum()
    loss.backward()

    pp = port.params_from_numpy(sd, requires_grad=True)
    xr = torch.from_numpy(batch["inputs"]).clone().requires_grad_(True)
    cr = torch.from_numpy(batch["case_params"]).clone().requires_grad_(True)
    mr = torch.from_numpy(batch["mask"])
    cur, ref_loss = xr, 0.0
    for s in range(steps):
        cur = port.forward(pp, cur, cr, mr, round_fn=_round_fn(act))["preds"]
        ref_loss = ref_loss + (cur * weights[s]).sum()
    ref_loss.backward()
    tol = _tol(act)
    assert _rel(x0.grad, xr.grad) < tol, _rel(x0.grad, xr.grad)
    assert _rel(cp.grad, cr.grad) < tol, _rel(cp.grad, cr.grad)
    for k, v in m.named_parameters():
        assert _rel(v.grad, pp[k].grad) < tol, (k, _rel(v.grad, pp[k].grad))


def test_mask_gradients_raise_and_no_grad_takes_the_inference_path():
    from cfdbench_b200 import synth
    p = 5
    sd = synth.make_state_dict(91, n_params=p, spectral_gain=50.0)
    batch = synth.make_batch(92, 2, "cavity")
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    m = _model(sd, p, "float32")
    with pytest.raises(NotImplementedError, match="mask"):
        m(inputs=tb["inputs"], case_params=tb["case_params"], mask=tb["mask"].clone().requires_grad_(True))
    for prm in m.parameters():   # a frozen model does not hide the error either
        prm.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="mask"):
        m(inputs=tb["inputs"], case_params=tb["case_params"], mask=tb["mask"].clone().requires_grad_(True))

    def no_training_path(*a, **k):
        raise AssertionError("training path taken without grad mode")
    m._native_forward_train = no_training_path
    x = tb["inputs"].clone().requires_grad_(True)
    cp = tb["case_params"].clone().requires_grad_(True)
    for ctx in (torch.no_grad, torch.inference_mode):
        with ctx():
            y = m.generate(x, cp, tb["mask"])
        assert not y.requires_grad and y.grad_fn is None


def test_model_without_case_params():
    """p = 0: the (B, 0) case-parameter gradient is empty and the input gradient still matches the port."""
    from cfdbench_b200 import synth
    from oracle import fno_torch_port as port
    sd = synth.make_state_dict(101, n_params=0, spectral_gain=50.0)
    batch = synth.make_batch(102, 3, "cavity")
    batch["case_params"] = np.zeros((3, 0), np.float32)
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    m = _model(sd, 0, "float32").requires_grad_(False)
    x = tb["inputs"].clone().requires_grad_(True)
    cp = tb["case_params"].clone().requires_grad_(True)
    m(inputs=x, case_params=cp, mask=tb["mask"], label=tb["label"])["loss"]["nmse"].backward()
    assert cp.grad.shape == (3, 0)
    pp = port.params_from_numpy(sd)
    xr = torch.from_numpy(batch["inputs"]).clone().requires_grad_(True)
    o = port.forward(pp, xr, torch.from_numpy(batch["case_params"]), torch.from_numpy(batch["mask"]),
                     label=torch.from_numpy(batch["label"]))
    o["loss"]["nmse"].backward()
    assert _rel(x.grad, xr.grad) < 5e-5, _rel(x.grad, xr.grad)
