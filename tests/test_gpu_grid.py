"""Grid-generic fp32 path (fno_grid_*, fno_grid.cu) on the GPU: the 66x65 tube fixture of the reference, every kernel
against the float64 numpy oracle on grids that land on the partial-tile tails, the generic kernels at 64x64 against the
64x64 fp32 kernels, input gradients against autograd of the torch port, bit-reproducibility, a full batch, and the
reference's own scripts on a tiny tube set."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.special import erf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "grid", "tube_b2_66x65.npz")
REF_SRC = os.path.join(ROOT, "oracle", "_ref", "src")
GRIDS = [(66, 65), (65, 66), (24, 24), (128, 128), (40, 48)]
BATCHES = [1, 3, 70]


def _gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def _dgelu(x):
    return 0.5 * (1.0 + erf(x / np.sqrt(2.0))) + x * np.exp(-0.5 * x * x) / np.sqrt(2.0 * np.pi)


def _model(sd, p, **kw):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m


def _np(t):
    if torch.is_tensor(t):
        t = t.detach().cpu()
        return (torch.view_as_real(t) if t.is_complex() else t).double().numpy()
    t = np.asarray(t)
    return np.stack([t.real, t.imag], -1) if np.iscomplexobj(t) else t.astype(np.float64)


def _rel(a, ref) -> float:
    a, ref = _np(a), _np(ref)
    return float(np.linalg.norm(a - ref) / np.linalg.norm(ref))


def _per_sample_rel(a, ref):
    a = a.detach().cpu().double().numpy().reshape(a.shape[0], -1)
    ref = np.asarray(ref, np.float64).reshape(a.shape[0], -1)
    return np.linalg.norm(a - ref, axis=1) / np.linalg.norm(ref, axis=1)


def _golden():
    from cfdbench_b200 import synth
    g = np.load(GOLD)
    p = synth.n_case_params(str(g["problem"]))
    sd = synth.make_state_dict(int(g["weight_seed"]), n_params=p, spectral_gain=float(g["spectral_gain"]))
    batch = synth.make_batch(int(g["batch_seed"]), g["preds"].shape[0], str(g["problem"]))
    return g, sd, batch, p


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ tube fixture
def test_tube_fixture_forward_loss_grads_and_rollouts():
    g, sd, batch, p = _golden()
    m = _model(sd, p)
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    out = m(**tb)
    assert _per_sample_rel(out["preds"], g["preds"]).max() <= 1e-5
    for i, k in enumerate(("mse", "rmse", "mae", "nmse")):
        assert abs(out["loss"][k].item() - g["loss"][i]) <= 1e-5 * abs(g["loss"][i]), k
    out["loss"]["nmse"].backward()
    grads = dict(m.named_parameters())
    for k in g.files:
        if k.startswith("grad::"):
            name = k[len("grad::"):]
            assert _rel(grads[name].grad, g[k]) <= 5e-5, name
        elif k.startswith("gradslice::"):
            name = k[len("gradslice::"):]
            gs = grads[name].grad.detach().cpu().numpy()[:, :, ::4, ::4]
            assert np.linalg.norm(gs - g[k]) <= 5e-5 * float(g["gradnorm::" + name]), name
    steps = int(g["steps"])
    seq = m.generate_many(tb["inputs"], tb["case_params"], tb["mask"], steps)
    host = m.generate_many(torch.from_numpy(batch["inputs"]), torch.from_numpy(batch["case_params"]),
                           torch.from_numpy(batch["mask"]), steps)
    for s in range(steps):
        assert seq[s].is_cuda and not host[s].is_cuda and host[s].is_pinned()
        assert _per_sample_rel(seq[s], g["rollout"][s]).max() <= 2e-5, s
        assert _per_sample_rel(host[s], g["rollout"][s]).max() <= 2e-5, s
    assert torch.equal(seq[-1].cpu(), host[-1])


# ------------------------------------------------------------------------------------------------ kernel by kernel
def _weights_struct(sd, p, gh, gw, keep):
    from cfdbench_b200 import _lib
    t = {k: torch.from_numpy(v).cuda() for k, v in sd.items() if not np.iscomplexobj(v)}
    gx = torch.tensor(np.linspace(0, 1, gh), dtype=torch.float).cuda()
    gy = torch.tensor(np.linspace(0, 1, gw), dtype=torch.float).cuda()
    keep += [t, gx, gy]
    w = _lib.FnoWeights()
    w.n_layers, w.n_case_params = 4, p
    w.fc0_w, w.fc0_b = t["fc0.weight"].data_ptr(), t["fc0.bias"].data_ptr()
    w.fc1_w, w.fc1_b = t["fc1.weight"].data_ptr(), t["fc1.bias"].data_ptr()
    w.fc2_w, w.fc2_b = t["fc2.weight"].data_ptr(), t["fc2.bias"].data_ptr()
    w.gx, w.gy = gx.data_ptr(), gy.data_ptr()
    return w


def _rand(rng, *shape):
    return rng.standard_normal(shape).astype(np.float32)


@pytest.mark.parametrize("b", BATCHES)
@pytest.mark.parametrize("gh,gw", GRIDS)
def test_lift_kernel(gh, gw, b):
    from cfdbench_b200 import _lib, synth
    from oracle import fno_numpy as onp
    lib, rng, keep = _lib.load(), np.random.default_rng(gh * 1000 + gw + b), []
    sd = synth.make_state_dict(5, n_params=8)
    w = _weights_struct(sd, 8, gh, gw, keep)
    x, cp, mk = _rand(rng, b, 2, gh, gw), _rand(rng, b, 8), (rng.random((b, gh, gw)) > 0.2).astype(np.float32)
    xg, cg, mg = (torch.from_numpy(t).cuda() for t in (x, cp, mk))
    out = torch.empty(b, 32, gh, gw, device="cuda")
    _lib.check(lib.fno_grid_lift_fwd(xg.data_ptr(), mg.data_ptr(), cg.data_ptr(), C.byref(w), out.data_ptr(), b, gh, gw, _s()),
               "lift")
    ref = onp.conv1x1(onp.lift_features(x, cp, mk), sd["fc0.weight"], sd["fc0.bias"])
    e = _rel(out, ref)
    assert e < 1e-6, e


@pytest.mark.parametrize("b", BATCHES)
@pytest.mark.parametrize("gh,gw", GRIDS)
def test_dft_kernel(gh, gw, b):
    from cfdbench_b200 import _lib
    from oracle import fno_numpy as onp
    lib, rng = _lib.load(), np.random.default_rng(gh * 1000 + gw + b)
    x = _rand(rng, b, 32, gh, gw)
    xm = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
    xg = torch.from_numpy(x).cuda()
    _lib.check(lib.fno_grid_spectral_dft_fwd(xg.data_ptr(), xm.data_ptr(), b, gh, gw, 0.5, 2.0, _s()), "dft")
    ref = onp.spectral_modes(x, 12, 12)      # (B, 32, 24, 12)
    ref[..., 0] *= 0.5
    ref[..., 1:] *= 2.0
    got = xm.cpu().numpy().reshape(24, 12, b, 32).transpose(2, 3, 0, 1)
    assert np.linalg.norm(got - ref) / np.linalg.norm(ref) < 2e-6


@pytest.mark.parametrize("b", BATCHES)
@pytest.mark.parametrize("gh,gw", GRIDS)
def test_inv_kx_and_block_out_kernels(gh, gw, b):
    from cfdbench_b200 import _lib
    from oracle import fno_numpy as onp
    lib, rng = _lib.load(), np.random.default_rng(gh * 1000 + gw + b)
    y = (rng.standard_normal((b, 32, 24, 12)) + 1j * rng.standard_normal((b, 32, 24, 12))) * 50.0
    ym = torch.from_numpy(np.ascontiguousarray(y.transpose(2, 3, 0, 1).reshape(288, b, 32), dtype=np.complex64)).cuda()
    x = _rand(rng, b, 32, gh, gw)
    wt = (_rand(rng, 32, 32) / 6).astype(np.float32)
    bias = _rand(rng, 32)
    pre_in = _rand(rng, b, 32, gh, gw)
    z = torch.empty(b, gh, 24, 32, device="cuda")
    inv = 1.0 / (gh * gw)
    _lib.check(lib.fno_grid_spectral_inv_kx(ym.data_ptr(), z.data_ptr(), b, gh, gw, inv, 2 * inv, _s()), "inv_kx")
    y64 = ym.cpu().numpy().reshape(24, 12, b, 32).transpose(2, 3, 0, 1).astype(np.complex128)
    spec = onp.spectral_inverse(y64, gh, gw, 12, 12)
    conv = np.einsum("io,bihw->bohw", wt.astype(np.float64), x.astype(np.float64))
    xg, pg = torch.from_numpy(x).cuda(), torch.from_numpy(pre_in).cuda()
    wg, bg = torch.from_numpy(wt).cuda(), torch.from_numpy(bias).cuda()
    for epi in range(4):
        out = torch.empty(b, 32, gh, gw, device="cuda")
        pre = torch.empty(b, 32, gh, gw, device="cuda")
        use_bias = epi in (0, 1)
        _lib.check(lib.fno_grid_block_out(epi, z.data_ptr(), xg.data_ptr(), wg.data_ptr(), bg.data_ptr() if use_bias else None,
                                          out.data_ptr(), pre.data_ptr(), pg.data_ptr(), b, gh, gw, _s()), "block_out")
        v = spec + conv + (bias.astype(np.float64)[None, :, None, None] if use_bias else 0.0)
        ref = {0: _gelu(v), 1: _gelu(v), 2: v * _dgelu(pre_in.astype(np.float64)), 3: v}[epi]
        e = _rel(out, ref)
        assert e < 2e-6, (epi, e)
        if epi == 1:
            e = _rel(pre, v)
            assert e < 2e-6, e


@pytest.mark.parametrize("b", BATCHES)
@pytest.mark.parametrize("gh,gw", GRIDS)
def test_projection_and_projection_backward_kernels(gh, gw, b):
    from cfdbench_b200 import _lib, synth
    lib, rng, keep = _lib.load(), np.random.default_rng(gh * 1000 + gw + b), []
    sd = synth.make_state_dict(6, n_params=5)
    w = _weights_struct(sd, 5, gh, gw, keep)
    a = _rand(rng, b, 32, gh, gw)
    pre = _rand(rng, b, 32, gh, gw)
    mk = (rng.random((b, gh, gw)) > 0.2).astype(np.float32)
    dp = _rand(rng, b, 2, gh, gw)
    ag, pg, mg, dg = (torch.from_numpy(t).cuda() for t in (a, pre, mk, dp))
    preds = torch.empty(b, 2, gh, gw, device="cuda")
    _lib.check(lib.fno_grid_project_fwd(ag.data_ptr(), mg.data_ptr(), C.byref(w), preds.data_ptr(), b, gh, gw, _s()), "proj")
    w1 = sd["fc1.weight"].reshape(128, 32).astype(np.float64)
    w2 = sd["fc2.weight"].reshape(2, 128).astype(np.float64)
    z1 = np.einsum("ji,bihw->bjhw", w1, a.astype(np.float64)) + sd["fc1.bias"].astype(np.float64)[None, :, None, None]
    h1 = _gelu(z1)
    raw = np.einsum("cj,bjhw->bchw", w2, h1) + sd["fc2.bias"].astype(np.float64)[None, :, None, None]
    assert _rel(preds, raw * mk[:, None]) < 2e-6

    dpre = torch.empty(b, 32, gh, gw, device="cuda")
    dz1 = torch.empty(min(b, _lib.BWD_CHUNK), 128, gh, gw, device="cuda")
    part = torch.empty(lib.fno_grid_bwd_partials_bytes(gh, gw), dtype=torch.uint8, device="cuda")
    g = [torch.empty(n, device="cuda") for n in (128 * 32, 128, 2 * 128, 2)]
    _lib.check(lib.fno_grid_project_bwd(ag.data_ptr(), dg.data_ptr(), mg.data_ptr(), pg.data_ptr(), C.byref(w),
                                        dpre.data_ptr(), dz1.data_ptr(), part.data_ptr(), *[t.data_ptr() for t in g],
                                        b, gh, gw, _s()), "proj_bwd")
    graw = dp.astype(np.float64) * mk[:, None]
    gz1 = np.einsum("cj,bchw->bjhw", w2, graw) * _dgelu(z1)
    ga = np.einsum("ji,bjhw->bihw", w1, gz1)
    assert _rel(dpre, ga * _dgelu(pre.astype(np.float64))) < 2e-6
    assert _rel(g[0].view(128, 32), np.einsum("bjhw,bihw->ji", gz1, a.astype(np.float64))) < 2e-6
    assert _rel(g[1], gz1.sum(axis=(0, 2, 3))) < 2e-6
    assert _rel(g[2].view(2, 128), np.einsum("bchw,bjhw->cj", graw, h1)) < 2e-6
    assert _rel(g[3], graw.sum(axis=(0, 2, 3))) < 2e-6


# ------------------------------------------------------------------------------------------------ 64x64 cross-check
@pytest.mark.parametrize("problem", ["cavity", "cylinder"])
def test_generic_path_at_64_matches_the_64x64_kernels(problem):
    from cfdbench_b200 import synth
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(81, n_params=p, spectral_gain=100.0)
    batch = synth.make_batch(82, 37, problem)
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    res = []
    for generic in (False, True):
        m = _model(sd, p)
        m.generic_grid_at_64 = generic
        out = m(**tb)
        out["loss"]["nmse"].backward()
        with torch.no_grad():
            roll = m.generate_many(tb["inputs"], tb["case_params"], tb["mask"], 2)
        res.append((out["preds"].detach(), {k: v.grad.detach().clone() for k, v in m.named_parameters()}, roll))
    (p_fast, g_fast, r_fast), (p_gen, g_gen, r_gen) = res
    e = _per_sample_rel(p_gen, p_fast.cpu().numpy()).max()
    assert e <= 1e-5, e
    e = _per_sample_rel(r_gen[0], r_fast[0].cpu().numpy()).max()
    assert e <= 1e-5, e
    e = _per_sample_rel(r_gen[1], r_fast[1].cpu().numpy()).max()   # the second step feeds back both paths' 1e-5 errors
    assert e <= 5e-5, e
    for k in g_fast:
        e = _rel(g_gen[k], g_fast[k])
        assert e <= 5e-5, (k, e)


# ------------------------------------------------------------------------------------------------ input gradients
def _port_step(sd, batch, want_inputs=True):
    from oracle import fno_torch_port as port
    pp = port.params_from_numpy(sd, requires_grad=True)
    cb = {k: torch.from_numpy(v) for k, v in batch.items()}
    xr = cb["inputs"].clone().requires_grad_(want_inputs)
    cr = cb["case_params"].clone().requires_grad_(want_inputs)
    o = port.forward(pp, xr, cr, cb["mask"], label=cb["label"])
    o["loss"]["nmse"].backward()
    return xr.grad, cr.grad, {k: v.grad for k, v in pp.items()}


def _step(m, tb, inputs_grad):
    x = tb["inputs"].clone().requires_grad_(inputs_grad)
    cp = tb["case_params"].clone().requires_grad_(inputs_grad)
    m.zero_grad(set_to_none=True)
    out = m(inputs=x, case_params=cp, mask=tb["mask"], label=tb["label"])
    out["loss"]["nmse"].backward()
    return x.grad, cp.grad, {k: (None if v.grad is None else v.grad.detach().clone()) for k, v in m.named_parameters()}


def test_input_gradients_frozen_model_and_reproducibility():
    from cfdbench_b200 import synth
    sd = synth.make_state_dict(91, n_params=5, spectral_gain=50.0)
    batch = synth.make_batch(92, 6, "tube")
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    m = _model(sd, 5)
    _, _, g_params = _step(m, tb, False)
    d_in, d_cp, g_all = _step(m, tb, True)
    d_in2, d_cp2, g_all2 = _step(m, tb, True)
    assert torch.equal(d_in, d_in2) and torch.equal(d_cp, d_cp2)
    for k in g_params:
        assert torch.equal(g_params[k], g_all[k]), k       # input gradients do not change parameter gradients by a bit
        assert torch.equal(g_all[k], g_all2[k]), k         # fixed-order reductions: bit-identical over runs
    xr, cr, gp = _port_step(sd, batch)
    assert _rel(d_in, xr) <= 5e-5 and _rel(d_cp, cr) <= 5e-5
    for k in g_params:
        assert _rel(g_all[k], gp[k]) <= 5e-5, k
    # frozen model: data-only backward
    for prm in m.parameters():
        prm.requires_grad_(False)
    d_in3, d_cp3, g_none = _step(m, tb, True)
    assert all(v is None for v in g_none.values())
    assert _rel(d_in3, xr) <= 5e-5 and _rel(d_cp3, cr) <= 5e-5


def test_unrolled_three_step_generate_chain_b70():
    from cfdbench_b200 import synth
    from oracle import fno_torch_port as port
    sd = synth.make_state_dict(93, n_params=5, spectral_gain=50.0)
    batch = synth.make_batch(94, 70, "tube")
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    m = _model(sd, 5)
    x = tb["inputs"].clone().requires_grad_(True)
    cur = x
    for _ in range(3):
        cur = m.generate(cur, tb["case_params"], tb["mask"])
    loss = (cur * tb["label"]).sum()
    loss.backward()
    pp = port.params_from_numpy(sd, requires_grad=True)
    cb = {k: torch.from_numpy(v) for k, v in batch.items()}
    xr = cb["inputs"].clone().requires_grad_(True)
    c = xr
    for _ in range(3):
        c = port.forward(pp, c, cb["case_params"], cb["mask"])["preds"]
    (c * cb["label"]).sum().backward()
    assert _rel(cur, c) <= 2e-5
    assert _rel(x.grad, xr.grad) <= 5e-5
    for k, v in m.named_parameters():
        assert _rel(v.grad, pp[k].grad) <= 5e-5, k


# ------------------------------------------------------------------------------------------------ full batch
def test_full_batch_properties_b256():
    from cfdbench_b200 import synth
    from oracle import fno_numpy as onp
    sd = synth.make_state_dict(95, n_params=5, spectral_gain=100.0)
    batch = synth.make_batch(96, 256, "dam")
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    m = _model(sd, 5)
    with torch.no_grad():
        y = m.generate(tb["inputs"], tb["case_params"], tb["mask"])
    idx = [0, 77, 128, 255]
    ref = onp.fno_forward(sd, batch["inputs"][idx], batch["case_params"][idx], batch["mask"][idx])["preds"]
    assert _per_sample_rel(y[idx], ref).max() <= 1e-5
    with torch.no_grad():   # samples are independent of their batch mates
        y1 = m.generate(tb["inputs"][77:78], tb["case_params"][77:78], tb["mask"][77:78])
    assert _rel(y1, y[77:78].cpu().numpy()) <= 1e-6
    assert torch.isfinite(y).all() and float((y * (1 - tb["mask"])).abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ reference scripts
def _make_tiny_tube(out_dir, n_cases=(4, 3, 3), frames=6, seed=0):
    """Tube cases in the reference's on-disk format (src/dataset/tube.py:15-50): u, v (T, 64, 64) float32 + case.json."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, 64), np.linspace(0, 1, 64), indexing="ij")
    for sub, n in zip(("prop", "bc", "geo"), n_cases):
        for c in range(n):
            d = os.path.join(out_dir, "tube", sub, f"case{c:04d}")
            os.makedirs(d, exist_ok=True)
            a, b, ph = rng.uniform(0.5, 2.0, 3)
            u = np.stack([np.sin(2 * np.pi * (a * xx + 0.07 * t)) * np.cos(np.pi * b * yy + ph) * (1 + 0.1 * t)
                          for t in range(frames)]).astype(np.float32)
            v = np.stack([-np.cos(2 * np.pi * (a * xx + 0.07 * t)) * np.sin(np.pi * b * yy + ph) * (1 + 0.1 * t)
                          for t in range(frames)]).astype(np.float32)
            np.save(os.path.join(d, "u.npy"), u)
            np.save(os.path.join(d, "v.npy"), v)
            with open(os.path.join(d, "case.json"), "w") as f:
                json.dump({"vel_in": float(rng.uniform(0.1, 1.0)), "density": float(rng.uniform(1, 10)),
                           "viscosity": float(rng.uniform(1e-3, 1e-2)), "height": 0.1, "width": 1.0}, f)
    return out_dir


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF_SRC, "models", "fno")),
                    reason="oracle/_ref/src (installed by __graft_entry__.build()) is not present")
def test_reference_scripts_run_unchanged_on_tube(tmp_path):
    src = str(tmp_path / "ref" / "src")
    shutil.copytree(REF_SRC, src)
    for root, dirs, files in os.walk(src):
        os.chmod(root, 0o755)
        for f in files:
            os.chmod(os.path.join(root, f), 0o644)
    data = _make_tiny_tube(str(tmp_path / "data"))
    out = str(tmp_path / "result")
    env = {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), "PYTHONDONTWRITEBYTECODE": "1"}
    common = ["--model", "fno", "--data_name", "tube_prop_bc_geo", "--loss_name", "nmse", "--lr", "0.001",
              "--data_dir", data, "--output_dir", out]

    def run(script, extra):
        cmd = [sys.executable, "-m", "cfdbench_b200.runner", src, script, "--stub-missing"] + common + extra
        return subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)

    r = run("train_auto.py", ["--num_epochs", "2", "--batch_size", "4", "--eval_batch_size", "2", "--eval_interval", "1",
                              "--log_interval", "2", "--mode", "train_test"])
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert "====== Training done ======" in r.stdout and "=== Testing done ===" in r.stdout
    run_dir = os.path.join(out, "auto", "tube_prop_bc_geo", "dt0.1", "fno", "lr0.001_d4_h32_m112_m212")
    assert os.path.isdir(run_dir), os.listdir(out)
    losses = json.load(open(os.path.join(run_dir, "train_losses.json")))
    assert len(losses) >= 2 and all(np.isfinite(losses))
    preds = torch.load(os.path.join(run_dir, "test", "preds.pt"))
    assert tuple(preds.shape[1:]) == (1, 66, 65)

    ckpt = os.path.join(run_dir, "ckpt-1", "model.pt")
    code = f"""
import sys, json, torch
sys.path.insert(0, {src!r}); sys.path.insert(0, {ROOT!r})
from models.fno.fno2d import Fno2d as Ref
from models.loss import loss_name_to_fn
sd = torch.load({ckpt!r}, map_location="cpu")
ref = Ref(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32, modes1=12, modes2=12)
ref.load_state_dict(sd); ref.eval()
from cfdbench_b200 import Fno2d, loss_name_to_fn as ours_loss
m = Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=ours_loss("nmse"), num_layers=4, hidden_dim=32, modes1=12, modes2=12)
m.load_state_dict(sd)
g = torch.Generator().manual_seed(0)
x = torch.randn(2, 2, 66, 65, generator=g); cp = torch.randn(2, 5, generator=g); mk = torch.ones(2, 1, 66, 65)
mk[:, :, :, 0] = 0; mk[:, :, 0] = 0; mk[:, :, -1] = 0
with torch.no_grad():
    a = ref.generate(inputs=x, case_params=cp, mask=mk)
    b = m.generate(x.cuda(), cp.cuda(), mk.cuda()).cpu()
print(json.dumps(dict(rel=float((a - b).norm() / a.norm()))))
"""
    r2 = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r2.returncode == 0, r2.stderr[-2000:]
    assert json.loads(r2.stdout.strip().splitlines()[-1])["rel"] < 1e-5

    r3 = run("test_multistep.py", [])
    assert r3.returncode == 0, (r3.stdout[-1500:], r3.stderr[-3000:])
    metrics = json.load(open(os.path.join(run_dir, "multistep_metrics.json")))
    assert len(metrics) > 0 and all(np.isfinite(m_["nmse"]) for m_ in metrics)
