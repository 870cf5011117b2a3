"""TEST INFRASTRUCTURE -- float64 numpy restatement of the reference FNO hot path.

This file is the parity *oracle*.  It is never imported by the product package
(`cfdbench_b200/`); only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline leg
may use it.  It restates, in closed form (truncated DFT sums evaluated as float64 matrix
products, no FFT library involved), what the reference computes with torch.fft / einsum / Conv2d:

* `spectral_conv`      <- reference src/models/fno/fno2d.py:59-82  (SpectralConv2d_fast.forward)
* `fno_block`          <- reference src/models/fno/fno2d.py:106-112 (FnoBlock.forward)
* `lift_features`      <- reference src/models/fno/fno2d.py:195-214, 244-255 (cat + get_coords)
* `fno_forward`        <- reference src/models/fno/fno2d.py:178-242 (Fno2d.forward)
* `mse_loss`           <- reference src/models/loss.py:22-37       (MseLoss.forward)
* `rollout`            <- reference src/models/fno/fno2d.py:257-295 (generate / generate_many)
* `spectral_conv_backward`, `fno_backward` <- what torch.autograd derives for the above
  (PyTorch complex-gradient convention: grad = dL/dRe + i dL/dIm).
* `fno_vjp`, `fno_vjp_saved` <- the same adjoint for any upstream d(preds), through the lift into the input frame and the
  case parameters; `fno_vjp_saved` takes the hidden activations of a forward pass as given (e.g. a GPU's saved ones).

Pinning: the reference ships no tests or golden vectors (SURVEY.md 4, 8c).  The oracle is pinned
against outputs of the reference module itself, generated in the build container by
`oracle/make_golden.py` and committed under `tests/golden/`.
"""
from __future__ import annotations

from math import erf, pi, sqrt

import numpy as np

_erf = np.vectorize(erf, otypes=[np.float64])


def gelu(x: np.ndarray) -> np.ndarray:
    """nn.GELU() default = exact erf form (reference fno2d.py:147)."""
    return 0.5 * x * (1.0 + _erf(x / sqrt(2.0)))


def dgelu(x: np.ndarray) -> np.ndarray:
    return 0.5 * (1.0 + _erf(x / sqrt(2.0))) + x * np.exp(-0.5 * x * x) / sqrt(2.0 * pi)


def kept_rows(h: int, m1: int) -> np.ndarray:
    """Row (kx) frequencies the reference keeps: [:m1] (weights1) then [-m1:] (weights2),
    reference fno2d.py:73-78."""
    return np.concatenate([np.arange(m1), np.arange(h - m1, h)])


def _dft_mats(h: int, w: int, m1: int, m2: int):
    kx = kept_rows(h, m1)
    fh = np.exp(-2j * pi * np.outer(kx, np.arange(h)) / h)  # (2*m1, H)
    fw = np.exp(-2j * pi * np.outer(np.arange(m2), np.arange(w)) / w)  # (m2, W)
    return fh, fw


def stack_weights(w1: np.ndarray, w2: np.ndarray) -> np.ndarray:
    """(Cin,Cout,m1,m2) x2 -> (Cin,Cout,2*m1,m2): weights1 serves rows 0..m1-1, weights2 rows
    H-m1..H-1 (reference fno2d.py:73-78)."""
    return np.concatenate([w1, w2], axis=2).astype(np.complex128)


def spectral_modes(x: np.ndarray, m1: int, m2: int) -> np.ndarray:
    """X[b,c,kxi,ky] = sum_{h,w} x e^{-2 pi i (kx h/H + ky w/W)} on the kept modes
    (= rfft2(x)[..., kept rows, :m2], reference fno2d.py:62,73-78)."""
    h, w = x.shape[-2:]
    fh, fw = _dft_mats(h, w, m1, m2)
    return np.einsum("kh,bchw,lw->bckl", fh, x.astype(np.float64), fw, optimize=True)


def spectral_inverse(y: np.ndarray, h: int, w: int, m1: int, m2: int,
                     c0: float | None = None, c1: float | None = None) -> np.ndarray:
    """irfft2 of the zero-padded spectrum (reference fno2d.py:65-81): inverse C2C along H, then
    C2R along W.  C2R semantics: only Re of the ky=0 column survives, ky>=1 columns count twice
    (their Hermitian mirror), the Nyquist column is never touched because m2 <= W/2.
    c0/c1 override the ky=0 / ky>=1 coefficients (used by the adjoint)."""
    fh, fw = _dft_mats(h, w, m1, m2)
    c = np.full(m2, 2.0 / (h * w) if c1 is None else c1)
    c[0] = 1.0 / (h * w) if c0 is None else c0
    z = np.einsum("kh,bokl->bohl", np.conj(fh), y, optimize=True)  # (B,O,H,m2) complex
    return np.einsum("bohl,lw->bohw", z * c, np.conj(fw), optimize=True).real


def spectral_conv(x: np.ndarray, w1: np.ndarray, w2: np.ndarray) -> np.ndarray:
    """SpectralConv2d_fast.forward (reference fno2d.py:59-82)."""
    m1, m2 = w1.shape[2:]
    wt = stack_weights(w1, w2)
    xm = spectral_modes(x, m1, m2)
    ym = np.einsum("bikl,iokl->bokl", xm, wt, optimize=True)
    return spectral_inverse(ym, x.shape[-2], x.shape[-1], m1, m2)


def conv1x1(x: np.ndarray, weight: np.ndarray, bias: np.ndarray) -> np.ndarray:
    wm = weight.reshape(weight.shape[0], weight.shape[1]).astype(np.float64)
    return np.einsum("oi,bihw->bohw", wm, x, optimize=True) + bias.astype(np.float64)[None, :, None, None]


def fno_block(x: np.ndarray, sd: dict, l: int, return_pre: bool = False):
    """FnoBlock.forward (reference fno2d.py:106-112): GELU(spectral(x) + w0(x)); the reference
    passes act_fn to every block, so GELU is applied on the last block too (fno2d.py:160-171)."""
    pre = spectral_conv(x, sd[f"blocks.{l}.conv0.weights1"], sd[f"blocks.{l}.conv0.weights2"]) \
        + conv1x1(x, sd[f"blocks.{l}.w0.weight"], sd[f"blocks.{l}.w0.bias"])
    return (gelu(pre), pre) if return_pre else gelu(pre)


def lift_features(inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray | None) -> np.ndarray:
    """Channel assembly [u, v, mask, x, y, params...] (reference fno2d.py:195-214); coordinates
    from get_coords (fno2d.py:244-255): x = linspace(0,1,H) along dim -2, y = linspace(0,1,W)
    along dim -1, built in float64 then cast to float32 by the reference."""
    b, _, h, w = inputs.shape
    if mask is None:
        mask = np.ones((b, 1, h, w))
    elif mask.ndim == 3:
        mask = mask[:, None]
    gx = np.linspace(0, 1, h).astype(np.float32).astype(np.float64).reshape(1, 1, h, 1)
    gy = np.linspace(0, 1, w).astype(np.float32).astype(np.float64).reshape(1, 1, 1, w)
    feats = [inputs.astype(np.float64), mask.astype(np.float64),
             np.broadcast_to(gx, (b, 1, h, w)), np.broadcast_to(gy, (b, 1, h, w)),
             np.broadcast_to(case_params.astype(np.float64)[:, :, None, None], (b, case_params.shape[1], h, w))]
    return np.concatenate(feats, axis=1)


def num_layers(sd: dict) -> int:
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))


def bf16_round(x: np.ndarray) -> np.ndarray:
    """Round to the nearest bf16 value (ties to even), result as float64."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    u = (u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return u.view(np.float32).astype(np.float64)


def fno_forward(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray | None = None,
                label: np.ndarray | None = None, normalize: bool = True, return_acts: bool = False,
                round_fn=None):
    """Fno2d.forward (reference fno2d.py:178-242).  Returns {"preds", ["loss"], ["acts"]}.
    `round_fn` (e.g. bf16_round) is applied to the hidden activations a_0..a_L, the tensors the CUDA path stores between
    kernels: float64 arithmetic + bf16 storage = a second, torch-independent "bf16-boundary oracle"."""
    b, _, h, w = inputs.shape
    m = np.ones((b, 1, h, w)) if mask is None else (mask[:, None] if mask.ndim == 3 else mask)
    m = m.astype(np.float64)
    rf = round_fn if round_fn is not None else (lambda t: t)
    a = rf(conv1x1(lift_features(inputs, case_params, m), sd["fc0.weight"], sd["fc0.bias"]))
    acts, pres = [a], []
    for l in range(num_layers(sd)):
        a, pre = fno_block(a, sd, l, return_pre=True)
        a = rf(a)
        acts.append(a)
        pres.append(pre)
    z1 = conv1x1(a, sd["fc1.weight"], sd["fc1.bias"])
    raw = conv1x1(gelu(z1), sd["fc2.weight"], sd["fc2.bias"])
    preds = raw * m
    out = {"preds": preds}
    if label is not None:
        out["loss"] = mse_loss(preds, label.astype(np.float64) * m, normalize)
    if return_acts:
        out["acts"], out["pres"], out["z1"] = acts, pres, z1
    return out


def mse_loss(preds: np.ndarray, labels: np.ndarray, normalize: bool = True) -> dict:
    """MseLoss.forward (reference src/models/loss.py:22-37): means over the whole batch tensor."""
    d = preds - labels
    mse = float(np.mean(d * d))
    res = {"mse": mse, "rmse": sqrt(mse), "mae": float(np.mean(np.abs(d)))}
    if normalize:
        res["nmse"] = mse / float(np.mean(labels * labels))
    return res


def rollout(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray, steps: int) -> list:
    """generate_many (reference fno2d.py:269-295): feed the (already masked) prediction back."""
    if inputs.ndim == 3:
        inputs, case_params, mask = inputs[None], case_params[None], mask[None]
    cur, outs = inputs.astype(np.float64), []
    for _ in range(steps):
        cur = fno_forward(sd, cur, case_params, mask)["preds"]
        outs.append(cur)
    return outs


def rel_l2(y: np.ndarray, ref: np.ndarray) -> float:
    """mean_b ||y-ref||_2 / ||ref||_2 (= LpLoss.rel, reference src/models/fno/utilities3.py:195-214)."""
    b = y.shape[0]
    d = np.linalg.norm((y.astype(np.float64) - ref).reshape(b, -1), axis=1)
    n = np.linalg.norm(ref.reshape(b, -1).astype(np.float64), axis=1)
    return float(np.mean(d / n))


# ----------------------------------------------------------------------------------------------
# Adjoint (what torch.autograd computes for the reference; SURVEY.md 8a "backward of the above")
# ----------------------------------------------------------------------------------------------

def spectral_conv_backward(x: np.ndarray, w1: np.ndarray, w2: np.ndarray, gy: np.ndarray):
    """Returns (gx, gw1, gw2) for y = spectral_conv(x, w1, w2) and upstream gradient gy."""
    m1, m2 = w1.shape[2:]
    h, w = x.shape[-2:]
    wt = stack_weights(w1, w2)
    xm = spectral_modes(x, m1, m2)
    c = np.full(m2, 2.0 / (h * w))
    c[0] = 1.0 / (h * w)
    g = spectral_modes(gy, m1, m2) * c  # grad wrt Y
    gxm = np.einsum("bokl,iokl->bikl", g, np.conj(wt), optimize=True)
    gwt = np.einsum("bikl,bokl->iokl", np.conj(xm), g, optimize=True)
    gx = spectral_inverse(gxm, h, w, m1, m2, c0=1.0, c1=1.0)
    return gx, gwt[:, :, :m1], gwt[:, :, m1:]


def fno_backward(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray,
                 label: np.ndarray, loss_key: str = "nmse") -> dict:
    """Gradients of loss[loss_key] w.r.t. every parameter (keys as in the state_dict)."""
    fwd = fno_forward(sd, inputs, case_params, mask, label, normalize=True, return_acts=True)
    b, _, h, w = inputs.shape
    m = (mask[:, None] if mask.ndim == 3 else mask).astype(np.float64)
    lab = label.astype(np.float64) * m
    preds, acts, pres, z1 = fwd["preds"], fwd["acts"], fwd["pres"], fwd["z1"]
    n = preds.size
    gp = 2.0 * (preds - lab) / n
    if loss_key == "nmse":
        gp = gp / float(np.mean(lab * lab))
    elif loss_key != "mse":
        raise ValueError(loss_key)
    grads: dict[str, np.ndarray] = {}
    graw = gp * m
    h1 = gelu(z1)
    w2m = sd["fc2.weight"].reshape(sd["fc2.weight"].shape[:2]).astype(np.float64)
    grads["fc2.weight"] = np.einsum("bchw,bjhw->cj", graw, h1, optimize=True)[:, :, None, None]
    grads["fc2.bias"] = graw.sum(axis=(0, 2, 3))
    gz1 = np.einsum("cj,bchw->bjhw", w2m, graw, optimize=True) * dgelu(z1)
    w1m = sd["fc1.weight"].reshape(sd["fc1.weight"].shape[:2]).astype(np.float64)
    grads["fc1.weight"] = np.einsum("bjhw,bihw->ji", gz1, acts[-1], optimize=True)[:, :, None, None]
    grads["fc1.bias"] = gz1.sum(axis=(0, 2, 3))
    ga = np.einsum("ji,bjhw->bihw", w1m, gz1, optimize=True)
    for l in reversed(range(num_layers(sd))):
        gpre = ga * dgelu(pres[l])
        x = acts[l]
        w0 = sd[f"blocks.{l}.w0.weight"].reshape(x.shape[1], x.shape[1]).astype(np.float64)
        grads[f"blocks.{l}.w0.weight"] = np.einsum("bohw,bihw->oi", gpre, x, optimize=True)[:, :, None, None]
        grads[f"blocks.{l}.w0.bias"] = gpre.sum(axis=(0, 2, 3))
        gxs, gw1, gw2 = spectral_conv_backward(x, sd[f"blocks.{l}.conv0.weights1"],
                                               sd[f"blocks.{l}.conv0.weights2"], gpre)
        grads[f"blocks.{l}.conv0.weights1"], grads[f"blocks.{l}.conv0.weights2"] = gw1, gw2
        ga = gxs + np.einsum("oi,bohw->bihw", w0, gpre, optimize=True)
    feats = lift_features(inputs, case_params, m)
    grads["fc0.weight"] = np.einsum("bohw,bihw->oi", ga, feats, optimize=True)[:, :, None, None]
    grads["fc0.bias"] = ga.sum(axis=(0, 2, 3))
    return grads


def _scipy_erf(x: np.ndarray) -> np.ndarray:
    from scipy.special import erf as sp_erf
    return sp_erf(x)


def fno_vjp_saved(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray, gpreds: np.ndarray,
                  acts: list, pres: list, erf=_scipy_erf, chunk: int = 32):
    """(parameter gradients, dL/dinputs, dL/dcase_params) for L = sum(gpreds * preds), float64, given the hidden
    activations a_0..a_L and the block pre-activations pre_0..pre_{L-1} of a forward pass.  With the saved tensors fixed
    the adjoint is a linear map of `gpreds`, so saved tensors of any forward -- this oracle's own, or a GPU's in either
    storage mode -- give a float64 reference of what a backward pass through them computes.  The lift is differentiated
    through a rounded a_0 and every GELU through its saved pre-activation (straight-through).  With
    a0 = fc0(cat[u, v, mask, x, y, params]) (reference fno2d.py:195-217) and ga = dL/da0,
        dL/du, dL/dv  = sum_o fc0_w[o][0|1] ga[b][o]          dL/dparams[b][j] = sum_o fc0_w[o][5+j] sum_hw ga[b][o].
    `erf` is the error function of the GELU terms; the projection runs in sample chunks of `chunk` to bound the size
    of its 128-channel temporaries."""
    def gelu_dgelu(x):
        e = erf(x / sqrt(2.0))
        return 0.5 * x * (1.0 + e), 0.5 * (1.0 + e) + x * np.exp(-0.5 * x * x) / sqrt(2.0 * pi)

    m = (mask[:, None] if mask.ndim == 3 else mask).astype(np.float64)
    a_last = acts[-1]
    grads: dict[str, np.ndarray] = {}
    w1m = sd["fc1.weight"].reshape(sd["fc1.weight"].shape[:2]).astype(np.float64)
    w2m = sd["fc2.weight"].reshape(sd["fc2.weight"].shape[:2]).astype(np.float64)
    g_w2 = np.zeros(w2m.shape)
    g_b2 = np.zeros(w2m.shape[0])
    g_w1 = np.zeros(w1m.shape)
    g_b1 = np.zeros(w1m.shape[0])
    ga = np.empty(a_last.shape)
    for b0 in range(0, a_last.shape[0], chunk):
        sl = slice(b0, b0 + chunk)
        a = np.asarray(a_last[sl], dtype=np.float64)
        h1, dh1 = gelu_dgelu(conv1x1(a, sd["fc1.weight"], sd["fc1.bias"]))
        graw = gpreds[sl].astype(np.float64) * m[sl]
        g_w2 += np.einsum("bchw,bjhw->cj", graw, h1, optimize=True)
        g_b2 += graw.sum(axis=(0, 2, 3))
        gz1 = np.einsum("cj,bchw->bjhw", w2m, graw, optimize=True) * dh1
        g_w1 += np.einsum("bjhw,bihw->ji", gz1, a, optimize=True)
        g_b1 += gz1.sum(axis=(0, 2, 3))
        ga[sl] = np.einsum("ji,bjhw->bihw", w1m, gz1, optimize=True)
    grads["fc2.weight"], grads["fc2.bias"] = g_w2[:, :, None, None], g_b2
    grads["fc1.weight"], grads["fc1.bias"] = g_w1[:, :, None, None], g_b1
    for l in reversed(range(num_layers(sd))):
        gpre = ga * gelu_dgelu(np.asarray(pres[l], dtype=np.float64))[1]
        x = np.asarray(acts[l], dtype=np.float64)
        w0 = sd[f"blocks.{l}.w0.weight"].reshape(x.shape[1], x.shape[1]).astype(np.float64)
        grads[f"blocks.{l}.w0.weight"] = np.einsum("bohw,bihw->oi", gpre, x, optimize=True)[:, :, None, None]
        grads[f"blocks.{l}.w0.bias"] = gpre.sum(axis=(0, 2, 3))
        gxs, gw1, gw2 = spectral_conv_backward(x, sd[f"blocks.{l}.conv0.weights1"],
                                               sd[f"blocks.{l}.conv0.weights2"], gpre)
        grads[f"blocks.{l}.conv0.weights1"], grads[f"blocks.{l}.conv0.weights2"] = gw1, gw2
        ga = gxs + np.einsum("oi,bohw->bihw", w0, gpre, optimize=True)
    feats = lift_features(inputs, case_params, m)
    grads["fc0.weight"] = np.einsum("bohw,bihw->oi", ga, feats, optimize=True)[:, :, None, None]
    grads["fc0.bias"] = ga.sum(axis=(0, 2, 3))
    w_lift = sd["fc0.weight"].reshape(sd["fc0.weight"].shape[:2]).astype(np.float64)   # [32][5+p]
    d_inputs = np.einsum("oc,bohw->bchw", w_lift[:, :inputs.shape[1]], ga, optimize=True)
    d_case_params = np.einsum("oj,bo->bj", w_lift[:, 5:], ga.sum(axis=(2, 3)), optimize=True)
    return grads, d_inputs, d_case_params


def fno_vjp(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray, gpreds: np.ndarray, erf=_scipy_erf):
    """fno_vjp_saved through this oracle's own float64 forward: the exact vector-Jacobian product of Fno2d."""
    fwd = fno_forward(sd, inputs, case_params, mask, return_acts=True)
    return fno_vjp_saved(sd, inputs, case_params, mask, gpreds, fwd["acts"], fwd["pres"], erf=erf)
