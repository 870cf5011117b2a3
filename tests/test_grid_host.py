"""Grid-generic path, host side: the oracles against the 66x65 tube fixture of the reference, the grid checks of the
module, and the fno_grid_* symbols of the library."""
import ctypes
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "grid", "tube_b2_66x65.npz")


def _golden():
    from cfdbench_b200 import synth
    g = np.load(GOLD)
    problem = str(g["problem"])
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(int(g["weight_seed"]), n_params=p, spectral_gain=float(g["spectral_gain"]))
    batch = synth.make_batch(int(g["batch_seed"]), g["preds"].shape[0], problem)
    return g, sd, batch, p


def _model(p=5, **kw):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    return Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                 modes1=12, modes2=12, device="cpu", **kw)


def test_tube_synth_batch_layout():
    from cfdbench_b200 import synth
    assert synth.grid("tube") == synth.grid("dam") == (66, 65)
    assert synth.grid("cavity") == synth.grid("cylinder") == (64, 64)
    b = synth.make_batch(1, 3, "dam")
    assert b["inputs"].shape == (3, 2, 66, 65) and b["mask"].shape == (3, 1, 66, 65) and b["case_params"].shape == (3, 5)
    m = b["mask"][0, 0]
    assert m[:, 0].sum() == 0 and m[0].sum() == 0 and m[-1].sum() == 0 and m[1:-1, 1:].min() == 1


def test_numpy_oracle_and_torch_port_reproduce_the_tube_fixture():
    from oracle import fno_numpy as onp
    from oracle import fno_torch_port as opt
    g, sd, batch, _ = _golden()
    assert g["preds"].shape == (2, 2, 66, 65)
    out = onp.fno_forward(sd, batch["inputs"], batch["case_params"], batch["mask"], batch["label"])
    assert onp.rel_l2(g["preds"], out["preds"]) < 2e-6
    for i, k in enumerate(("mse", "rmse", "mae", "nmse")):
        assert abs(out["loss"][k] - g["loss"][i]) < 1e-5 * abs(g["loss"][i])
    grads = onp.fno_backward(sd, batch["inputs"], batch["case_params"], batch["mask"], batch["label"])
    for k in g.files:
        if k.startswith("grad::"):
            name = k[len("grad::"):]
            assert np.linalg.norm(grads[name] - g[k]) / np.linalg.norm(g[k]) < 5e-5, name
        elif k.startswith("gradnorm::"):
            name = k[len("gradnorm::"):]
            assert abs(np.linalg.norm(grads[name]) - float(g[k])) < 5e-5 * float(g[k]), name
    roll = onp.rollout(sd, batch["inputs"], batch["case_params"], batch["mask"], int(g["steps"]))
    for s in range(int(g["steps"])):
        assert onp.rel_l2(g["rollout"][s], roll[s]) < 1e-5, s

    pp = opt.params_from_numpy(sd)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    pout = opt.forward(pp, tb["inputs"], tb["case_params"], tb["mask"], tb["label"])
    np.testing.assert_array_equal(pout["preds"].detach().numpy(), g["preds"])   # the port is bit-exact on CPU


def test_grid_range_and_storage_checks():
    m = _model()
    cp = torch.zeros(2, 5)
    x, _, mk = m._prep_inputs(torch.zeros(2, 2, 66, 65), cp, torch.ones(2, 66, 65))
    assert x.shape == (2, 2, 66, 65) and mk.shape == (2, 1, 66, 65)
    for shape in [(23, 64), (64, 23), (129, 64), (64, 129), (16, 16)]:
        with pytest.raises(ValueError, match="grid"):
            m._prep_inputs(torch.zeros(2, 2, *shape), cp, None)
    with pytest.raises(ValueError, match="mask"):
        m._prep_inputs(torch.zeros(2, 2, 66, 65), cp, torch.ones(2, 64, 64))
    m16 = _model(act_dtype="bfloat16")
    with pytest.raises(ValueError, match="66x65"):
        m16._prep_inputs(torch.zeros(2, 2, 66, 65), cp, None)
    m16._prep_inputs(torch.zeros(2, 2, 64, 64), cp, None)   # bf16 storage stays available on 64x64


def test_cpu_model_has_no_fallback_on_any_grid():
    from cfdbench_b200 import _lib
    m = _model()
    with pytest.raises(_lib.FnoNativeError):
        m(torch.zeros(1, 2, 66, 65), torch.zeros(1, 5))
    with pytest.raises(_lib.FnoNativeError):
        m.generate_many(torch.zeros(2, 66, 65), torch.zeros(5), torch.ones(66, 65), 2)


def test_grid_symbols_and_size_helpers():
    from cfdbench_b200 import _lib, build
    path = build.build()
    lib = ctypes.CDLL(path)
    for name in ("fno_grid_act_bytes", "fno_grid_z_bytes", "fno_grid_bwd_partials_bytes", "fno_grid_lift_fwd",
                 "fno_grid_spectral_dft_fwd", "fno_grid_spectral_inv_kx", "fno_grid_block_out", "fno_grid_project_fwd",
                 "fno_grid_project_bwd", "fno_grid_forward", "fno_grid_rollout", "fno_grid_forward_train",
                 "fno_grid_backward"):
        assert hasattr(lib, name), name
    L = _lib.load()
    assert L.fno_grid_act_bytes(3, 66, 65) == 3 * 32 * 66 * 65 * 4
    assert L.fno_grid_z_bytes(3, 66) == 3 * 66 * 24 * 32 * 4
    assert L.fno_grid_bwd_partials_bytes(66, 65) > 0
    # an out-of-range grid is refused before anything touches the device
    st = L.fno_grid_forward(None, None, None, None, None, None, 1, 20, 65, None)
    assert st != 0 and b"outside the supported range" in L.fno_last_error()
