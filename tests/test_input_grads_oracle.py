"""The oracle's float64 vector-Jacobian product (`oracle.fno_numpy.fno_vjp` / `fno_vjp_saved`) for an arbitrary upstream
gradient, including the gradients w.r.t. the input frame and the case parameters -- the yardstick of Fno2d's input
gradients (fno_backward_inputs) and, fed a GPU's saved activations, of the training backward stage by stage
(tests/test_gpu_train_conditioned.py).  Its parameter gradients must reproduce the oracle's adjoint
(`oracle.fno_numpy.fno_backward`); checked here also against autograd of the fp32 torch port and against central
finite differences of the float64 forward."""
import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import fno_numpy as onp
from oracle import fno_torch_port as port
from oracle.fno_numpy import fno_vjp


def nmse_upstream(preds: np.ndarray, label: np.ndarray, mask: np.ndarray) -> np.ndarray:
    """d nmse / d preds as oracle.fno_numpy.fno_backward forms it."""
    m = (mask[:, None] if mask.ndim == 3 else mask).astype(np.float64)
    lab = label.astype(np.float64) * m
    return 2.0 * (preds - lab) / preds.size / float(np.mean(lab * lab))


def _case(problem: str, seed: int, batch: int = 2):
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(seed, n_params=p, spectral_gain=50.0)
    bt = synth.make_batch(seed + 1, batch, problem)
    gp = np.random.default_rng(seed + 2).standard_normal(bt["inputs"].shape).astype(np.float32)
    return sd, bt, gp


def _rel(a, ref) -> float:
    return float(np.linalg.norm(np.asarray(a) - ref) / np.linalg.norm(ref))   # float64 / complex128 difference


@pytest.mark.parametrize("problem", ["cavity", "cylinder"])
def test_vjp_parameter_gradients_equal_oracle_backward(problem):
    sd, bt, _ = _case(problem, 21)
    preds = onp.fno_forward(sd, bt["inputs"], bt["case_params"], bt["mask"])["preds"]
    grads, _, _ = fno_vjp(sd, bt["inputs"], bt["case_params"], bt["mask"], nmse_upstream(preds, bt["label"], bt["mask"]))
    ref = onp.fno_backward(sd, bt["inputs"], bt["case_params"], bt["mask"], bt["label"])
    assert set(grads) == set(ref)
    for k, v in ref.items():
        np.testing.assert_allclose(grads[k], v, rtol=1e-12, atol=1e-15 * float(np.abs(v).max()), err_msg=k)


def test_vjp_saved_with_the_oracles_own_activations_reproduces_oracle_backward():
    """fno_vjp_saved fed fno_forward's own a_0..a_L / pre_0..pre_{L-1} and the nmse upstream: fno_backward's gradients.
    Three samples in projection chunks of two (a ragged last chunk), the GELU terms through math.erf instead of scipy."""
    sd, bt, _ = _case("cylinder", 23, batch=3)
    fwd = onp.fno_forward(sd, bt["inputs"], bt["case_params"], bt["mask"], return_acts=True)
    gp = nmse_upstream(fwd["preds"], bt["label"], bt["mask"])
    grads, d_in, d_cp = onp.fno_vjp_saved(sd, bt["inputs"], bt["case_params"], bt["mask"], gp, fwd["acts"], fwd["pres"],
                                          erf=onp._erf, chunk=2)
    ref = onp.fno_backward(sd, bt["inputs"], bt["case_params"], bt["mask"], bt["label"])
    assert set(grads) == set(ref)
    for k, v in ref.items():
        np.testing.assert_allclose(grads[k], v, rtol=1e-12, atol=1e-12 * float(np.abs(v).max()), err_msg=k)
    _, d_in2, d_cp2 = fno_vjp(sd, bt["inputs"], bt["case_params"], bt["mask"], gp)
    np.testing.assert_allclose(d_in, d_in2, rtol=1e-12, atol=1e-12 * float(np.abs(d_in2).max()))
    np.testing.assert_allclose(d_cp, d_cp2, rtol=1e-12, atol=1e-12 * float(np.abs(d_cp2).max()))


@pytest.mark.parametrize("problem", ["cavity", "cylinder"])
def test_vjp_input_gradients_match_torch_port_autograd(problem):
    """cavity: p = 5, full mask; cylinder: p = 8, holed mask."""
    sd, bt, gp = _case(problem, 31)
    grads, d_in, d_cp = fno_vjp(sd, bt["inputs"], bt["case_params"], bt["mask"], gp)
    pp = port.params_from_numpy(sd, requires_grad=True)
    x = torch.from_numpy(bt["inputs"]).requires_grad_(True)
    cp = torch.from_numpy(bt["case_params"]).requires_grad_(True)
    out = port.forward(pp, x, cp, torch.from_numpy(bt["mask"]))["preds"]
    (out * torch.from_numpy(gp)).sum().backward()
    assert d_in.shape == x.shape and d_cp.shape == cp.shape
    assert _rel(x.grad.numpy(), d_in) < 5e-5
    assert _rel(cp.grad.numpy(), d_cp) < 5e-5
    for k, v in grads.items():
        assert _rel(pp[k].grad.numpy(), v) < 5e-5, k


@pytest.mark.parametrize("problem", ["cavity", "cylinder"])
def test_vjp_input_gradients_match_finite_differences(problem):
    """Central differences of the float64 forward on a few case parameters and input pixels (both channels, one in the
    cylinder's masked region too: the inputs enter the lift unmasked)."""
    sd, bt, gp = _case(problem, 41, batch=1)
    inputs = bt["inputs"].astype(np.float64)
    cps = bt["case_params"].astype(np.float64)
    gp64 = gp.astype(np.float64)
    _, d_in, d_cp = fno_vjp(sd, inputs, cps, bt["mask"], gp64)

    def loss(x, c):
        return float(np.sum(gp64 * onp.fno_forward(sd, x, c, bt["mask"])["preds"]))

    eps = 1e-4
    fd, an = [], []
    for j in range(0, cps.shape[1], 3):
        cp_p, cp_m = cps.copy(), cps.copy()
        cp_p[0, j] += eps
        cp_m[0, j] -= eps
        fd.append((loss(inputs, cp_p) - loss(inputs, cp_m)) / (2 * eps))
        an.append(d_cp[0, j])
    pix = [(0, 5, 7), (1, 40, 20), (0, 63, 0), (1, 0, 63)]
    if problem == "cylinder":
        pix.append((0, 0, 31))   # the first row is masked out of the prediction
    for c, h, w in pix:
        x_p, x_m = inputs.copy(), inputs.copy()
        x_p[0, c, h, w] += eps
        x_m[0, c, h, w] -= eps
        fd.append((loss(x_p, cps) - loss(x_m, cps)) / (2 * eps))
        an.append(d_in[0, c, h, w])
    fd, an = np.array(fd), np.array(an)
    assert np.all(np.abs(an) > 0)
    assert np.linalg.norm(fd - an) / np.linalg.norm(an) <= 1e-6, (fd, an)
    assert np.max(np.abs(fd - an) / np.abs(an)) <= 1e-5, (fd, an)
