"""TEST INFRASTRUCTURE -- float64 backpropagation through a K-step rollout of Fno2d, built on `oracle.fno_numpy`.

`fno_rollout_vjp` is the yardstick of `Fno2d.rollout`'s backward (fno_rollout_backward): the same sweep s = K-1 .. 0,
each step's vector-Jacobian product (`fno_vjp_saved` through a float64 forward of that step's input frame) taken with
the upstream gradient gpreds_seq[s] + carry, carry = dL/d(frame fed to step s+1).  Never imported by the product
package.
"""
from __future__ import annotations

import numpy as np

from .fno_numpy import _scipy_erf, fno_forward, fno_vjp_saved


def fno_rollout_vjp(sd: dict, inputs: np.ndarray, case_params: np.ndarray, mask: np.ndarray, gpreds_seq: np.ndarray,
                    frames=None, erf=_scipy_erf):
    """(parameter gradients, dL/dinputs, dL/dcase_params) for L = sum_s sum(gpreds_seq[s] * preds_s), float64, where
    preds_s = Fno2d(frame_s) and frame_0 = inputs.  `gpreds_seq`: (K, B, 2, H, W).

    frames = None: frame_s = preds_{s-1} of this oracle's own float64 rollout (the exact adjoint of the rollout).
    frames given ((K, B, 2, H, W) or a list of K frames, e.g. a GPU's predictions): frame_s = frames[s-1], so every step
    is linearised at the trajectory that was actually computed -- the conditioning that compares a backward pass with
    its own forward's frames rather than with a trajectory that has drifted away from them.  frames[K-1] is not used.
    Parameter and case-parameter gradients are summed over the steps (the parameters and the case parameters feed every
    step)."""
    steps = len(gpreds_seq)
    m = (mask[:, None] if mask.ndim == 3 else mask).astype(np.float64)
    x = [np.asarray(inputs, dtype=np.float64)]
    if frames is None:
        for s in range(steps - 1):
            x.append(fno_forward(sd, x[-1], case_params, m)["preds"])
    else:
        x += [np.asarray(frames[s], dtype=np.float64) for s in range(steps - 1)]
    grads: dict = {}
    d_cp = None
    carry = None
    for s in reversed(range(steps)):
        fwd = fno_forward(sd, x[s], case_params, m, return_acts=True)
        up = np.asarray(gpreds_seq[s], dtype=np.float64)
        if carry is not None:
            up = up + carry
        g, carry, dcp_s = fno_vjp_saved(sd, x[s], case_params, m, up, fwd["acts"], fwd["pres"], erf=erf)
        for k, v in g.items():
            grads[k] = v if k not in grads else grads[k] + v
        d_cp = dcp_s if d_cp is None else d_cp + dcp_s
    return grads, carry, d_cp
