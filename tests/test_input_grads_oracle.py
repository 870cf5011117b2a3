"""Float64 vector-Jacobian product of the FNO forward for an arbitrary upstream gradient, including the gradients w.r.t.
the input frame and the case parameters -- the yardstick of Fno2d's input gradients (fno_backward_inputs).  It extends
the oracle's adjoint (`oracle.fno_numpy.fno_backward`, whose parameter gradients it must reproduce) through the lift:
with a0 = fc0(cat[u, v, mask, x, y, params]) (reference fno2d.py:195-217) and ga = dL/da0,
    dL/du, dL/dv  = sum_o fc0_w[o][0|1] ga[b][o]          dL/dparams[b][j] = sum_o fc0_w[o][5+j] sum_hw ga[b][o].
Checked here against autograd of the fp32 torch port and against central finite differences of the float64 forward."""
import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import fno_numpy as onp
from oracle import fno_torch_port as port


def fno_vjp(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray, gpreds: np.ndarray):
    """(parameter gradients, dL/dinputs, dL/dcase_params) for L = sum(gpreds * preds), float64."""
    fwd = onp.fno_forward(sd, inputs, case_params, mask, return_acts=True)
    m = (mask[:, None] if mask.ndim == 3 else mask).astype(np.float64)
    acts, pres, z1 = fwd["acts"], fwd["pres"], fwd["z1"]
    grads = {}
    graw = gpreds.astype(np.float64) * m
    h1 = onp.gelu(z1)
    w2m = sd["fc2.weight"].reshape(sd["fc2.weight"].shape[:2]).astype(np.float64)
    grads["fc2.weight"] = np.einsum("bchw,bjhw->cj", graw, h1, optimize=True)[:, :, None, None]
    grads["fc2.bias"] = graw.sum(axis=(0, 2, 3))
    gz1 = np.einsum("cj,bchw->bjhw", w2m, graw, optimize=True) * onp.dgelu(z1)
    w1m = sd["fc1.weight"].reshape(sd["fc1.weight"].shape[:2]).astype(np.float64)
    grads["fc1.weight"] = np.einsum("bjhw,bihw->ji", gz1, acts[-1], optimize=True)[:, :, None, None]
    grads["fc1.bias"] = gz1.sum(axis=(0, 2, 3))
    ga = np.einsum("ji,bjhw->bihw", w1m, gz1, optimize=True)
    for l in reversed(range(onp.num_layers(sd))):
        gpre = ga * onp.dgelu(pres[l])
        x = acts[l]
        w0 = sd[f"blocks.{l}.w0.weight"].reshape(x.shape[1], x.shape[1]).astype(np.float64)
        grads[f"blocks.{l}.w0.weight"] = np.einsum("bohw,bihw->oi", gpre, x, optimize=True)[:, :, None, None]
        grads[f"blocks.{l}.w0.bias"] = gpre.sum(axis=(0, 2, 3))
        gxs, gw1, gw2 = onp.spectral_conv_backward(x, sd[f"blocks.{l}.conv0.weights1"],
                                                   sd[f"blocks.{l}.conv0.weights2"], gpre)
        grads[f"blocks.{l}.conv0.weights1"], grads[f"blocks.{l}.conv0.weights2"] = gw1, gw2
        ga = gxs + np.einsum("oi,bohw->bihw", w0, gpre, optimize=True)
    feats = onp.lift_features(inputs, case_params, m)
    grads["fc0.weight"] = np.einsum("bohw,bihw->oi", ga, feats, optimize=True)[:, :, None, None]
    grads["fc0.bias"] = ga.sum(axis=(0, 2, 3))
    w_lift = sd["fc0.weight"].reshape(sd["fc0.weight"].shape[:2]).astype(np.float64)   # [32][5+p]
    d_inputs = np.einsum("oc,bohw->bchw", w_lift[:, :inputs.shape[1]], ga, optimize=True)
    d_case_params = np.einsum("oj,bo->bj", w_lift[:, 5:], ga.sum(axis=(2, 3)), optimize=True)
    return grads, d_inputs, d_case_params


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
