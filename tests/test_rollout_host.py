"""CPU checks of `Fno2d.rollout`'s yardstick and native surface: the float64 backpropagation-through-time oracle
(`oracle.fno_rollout_numpy.fno_rollout_vjp`) against float64 torch autograd of a chained rollout, and the rollout
training entry points of the C ABI (present, argument checks answered with a status before any device work)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cfdbench_b200 import synth
from oracle.fno_rollout_numpy import fno_rollout_vjp


# ---------------------------------------------------------------- float64 torch restatement of the CPU port's forward
def _spectral64(x, w1, w2):
    """oracle.fno_torch_port.spectral_conv in complex128 (the port's spectrum buffer is complex64)."""
    m1, m2 = w1.shape[-2:]
    spec = torch.fft.rfft2(x)
    out = torch.zeros(x.shape[0], w1.shape[1], x.shape[-2], x.shape[-1] // 2 + 1, dtype=torch.complex128)
    out[:, :, :m1, :m2] = torch.einsum("bixy,ioxy->boxy", spec[:, :, :m1, :m2], w1)
    out[:, :, -m1:, :m2] = torch.einsum("bixy,ioxy->boxy", spec[:, :, -m1:, :m2], w2)
    return torch.fft.irfft2(out, s=(x.shape[-2], x.shape[-1]))


def _forward64(p, x, cp, mask):
    """oracle.fno_torch_port.forward in float64 (coordinates rounded to float32 first, as the reference builds them)."""
    b, _, h, w = x.shape
    gx = torch.tensor(np.linspace(0, 1, h).astype(np.float32), dtype=torch.float64).reshape(1, 1, h, 1).expand(b, 1, h, w)
    gy = torch.tensor(np.linspace(0, 1, w).astype(np.float32), dtype=torch.float64).reshape(1, 1, 1, w).expand(b, 1, h, w)
    feats = torch.cat([x, mask, gx, gy, cp[:, :, None, None].expand(b, cp.shape[1], h, w)], dim=1)
    a = F.conv2d(feats, p["fc0.weight"], p["fc0.bias"])
    depth = 1 + max(int(k.split(".")[1]) for k in p if k.startswith("blocks."))
    for l in range(depth):
        s = _spectral64(a, p[f"blocks.{l}.conv0.weights1"], p[f"blocks.{l}.conv0.weights2"])
        a = F.gelu(s + F.conv2d(a, p[f"blocks.{l}.w0.weight"], p[f"blocks.{l}.w0.bias"]))
    return F.conv2d(F.gelu(F.conv2d(a, p["fc1.weight"], p["fc1.bias"])), p["fc2.weight"], p["fc2.bias"]) * mask


def _case(seed, b, gh, gw, p, depth, steps):
    rng = np.random.default_rng(seed)
    sd = synth.make_state_dict(seed, n_params=p, depth=depth, spectral_gain=50.0)
    mask = np.ones((b, 1, gh, gw))
    mask[:, :, 0, :] = mask[:, :, :, gw - 1] = 0.0   # masked pixels: the frames fed back are masked predictions
    inputs = rng.standard_normal((b, 2, gh, gw))
    cp = rng.standard_normal((b, p))
    gseq = rng.standard_normal((steps, b, 2, gh, gw))
    return sd, inputs, cp, mask, gseq


def _rel(a, ref):
    return float(np.linalg.norm(np.asarray(a) - ref) / np.linalg.norm(ref))


@pytest.mark.parametrize("steps", [1, 3, 5])
@pytest.mark.parametrize("grid", [(64, 64), (66, 65)], ids=["64x64", "66x65"])
def test_rollout_vjp_matches_float64_autograd_of_the_chained_rollout(grid, steps):
    gh, gw = grid
    sd, inputs, cp, mask, gseq = _case(100 + steps, 2, gh, gw, 5, 2, steps)
    grads, d_in, d_cp = fno_rollout_vjp(sd, inputs, cp, mask, gseq)

    p = {k: torch.from_numpy(v.astype(np.complex128 if np.iscomplexobj(v) else np.float64)).requires_grad_(True)
         for k, v in sd.items()}
    x0 = torch.from_numpy(inputs).requires_grad_(True)
    c = torch.from_numpy(cp).requires_grad_(True)
    m = torch.from_numpy(mask)
    x, loss = x0, 0.0
    for s in range(steps):
        x = _forward64(p, x, c, m)
        loss = loss + (x * torch.from_numpy(gseq[s])).sum()
    loss.backward()

    assert set(grads) == set(p)
    errs = {k: _rel(p[k].grad.numpy(), v) for k, v in grads.items()}
    errs["d_inputs"] = _rel(x0.grad.numpy(), d_in)
    errs["d_case_params"] = _rel(c.grad.numpy(), d_cp)
    worst = max(errs, key=errs.get)
    print(f"\n[rollout-vjp {gh}x{gw} K={steps}] max rel {errs[worst]:.3g} ({worst})")
    assert errs[worst] <= 1e-12, (worst, errs[worst])


def test_rollout_vjp_with_its_own_frames_equals_the_exact_adjoint():
    """frames = the oracle's own trajectory gives the frames=None result; the last frame is not used."""
    from oracle import fno_numpy as onp
    sd, inputs, cp, mask, gseq = _case(7, 2, 64, 64, 3, 1, 3)
    traj = onp.rollout(sd, inputs, cp, mask, 3)
    traj[-1] = np.full_like(traj[-1], np.nan)
    a = fno_rollout_vjp(sd, inputs, cp, mask, gseq)
    b = fno_rollout_vjp(sd, inputs, cp, mask, gseq, frames=traj)
    for k in a[0]:
        np.testing.assert_array_equal(a[0][k], b[0][k], err_msg=k)
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[2], b[2])


# --------------------------------------------------------------------------------------- C ABI
@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib, build
    build.build()
    return _lib.load()


ROLLOUT_SYMBOLS = ["fno_rollout_forward_train", "fno_rollout_backward", "fno_grid_rollout_forward_train",
                   "fno_grid_rollout_backward"]


def test_rollout_symbols_are_exported_and_declared(lib):
    from cfdbench_b200 import _lib
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in ROLLOUT_SYMBOLS:
        assert name in _lib.SIGNATURES
        assert hasattr(raw, name)


def _status(lib, fn, *args):
    st = fn(*args)
    return st, lib.fno_last_error().decode()


def test_bad_steps_and_grids_return_a_status_before_device_work(lib):
    """All pointers NULL: a call that got as far as the device would fault, so a status proves the check came first."""
    n = None
    st, msg = _status(lib, lib.fno_rollout_forward_train, n, n, n, n, n, 0, n, n, 4, 0, n)
    assert st == 1 and "fno_rollout_forward_train" in msg
    st, msg = _status(lib, lib.fno_rollout_backward, n, n, n, n, n, n, n, 0, n, n, n, n, n, n, n, 4, 0, n)
    assert st == 1 and "fno_rollout_backward" in msg
    st, msg = _status(lib, lib.fno_rollout_backward, n, n, n, n, n, n, n, -3, n, n, n, n, n, n, n, 4, 0, n)
    assert st == 1
    st, msg = _status(lib, lib.fno_grid_rollout_forward_train, n, n, n, n, n, 0, n, n, 4, 66, 65, n)
    assert st == 1 and "fno_grid_rollout_forward_train" in msg
    st, msg = _status(lib, lib.fno_grid_rollout_backward, n, n, n, n, n, n, n, 0, n, n, n, n, n, n, n, 4, 66, 65, n)
    assert st == 1 and "fno_grid_rollout_backward" in msg
    for gh, gw in [(23, 64), (64, 129), (200, 200)]:
        st, msg = _status(lib, lib.fno_grid_rollout_forward_train, n, n, n, n, n, 3, n, n, 4, gh, gw, n)
        assert st == 3 and f"{gh}x{gw}" in msg
        st, msg = _status(lib, lib.fno_grid_rollout_backward, n, n, n, n, n, n, n, 3, n, n, n, n, n, n, n, 4, gh, gw, n)
        assert st == 3 and f"{gh}x{gw}" in msg


def test_rollout_backward_rejects_missing_buffers_before_device_work(lib):
    """steps > 1 needs the frames and the carry; something must be requested."""
    from cfdbench_b200 import _lib
    w, wb, sv, sc, ws = _lib.FnoWeights(), _lib.FnoWeightsBwd(), _lib.FnoTrainSaved(), _lib.FnoBwdScratch(), _lib.FnoWorkspace()
    w.n_layers, w.n_case_params = 4, 5
    fake = 4096   # never dereferenced: every call below must fail its checks first
    r = ctypes.byref
    # K = 2 without preds_seq / carry
    st, msg = _status(lib, lib.fno_rollout_backward, r(w), r(wb), fake, fake, fake, None, fake, 2, r(sv), None, r(sc), r(ws),
                      None, fake, None, 4, 0, None)
    assert st == 1 and "bad argument" in msg
    # no output requested
    st, msg = _status(lib, lib.fno_rollout_backward, r(w), r(wb), fake, fake, fake, fake, fake, 2, r(sv), None, r(sc), r(ws),
                      fake + 4096, None, None, 4, 0, None)
    assert st == 1 and "no output requested" in msg
    # null scratch
    st, msg = _status(lib, lib.fno_rollout_backward, r(w), r(wb), fake, fake, fake, fake, fake, 2, r(sv), None, r(sc), r(ws),
                      fake + 4096, fake + 8192, None, 4, 0, None)
    assert st == 1 and "scratch" in msg


def test_rollout_needs_a_cuda_model():
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    from cfdbench_b200._lib import FnoNativeError
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_name_to_fn("nmse"), num_layers=2, hidden_dim=32,
              modes1=12, modes2=12, device="cpu")
    with pytest.raises(FnoNativeError):
        m.rollout(torch.zeros(1, 2, 64, 64), torch.zeros(1, 5), torch.ones(1, 64, 64), 2)
