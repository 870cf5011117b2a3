"""GPU parity tests (run with `-m gpu` on an H100): every CUDA kernel and the whole model, called
through the C ABI / the drop-in module, against the oracles and the golden vectors generated from
the reference module.  Tolerance for fp32-storage mode is BASELINE.json's 1e-5 relative L2."""
import ctypes as C
import glob
import os

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import fno_numpy as onp
from oracle import fno_torch_port as opt

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

TOL = 1e-5  # relative L2, fp32 activation storage (north_star)
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()  # raises if the .so is missing: GPU tests must never pass on a fallback


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def make_model(sd, p, act_dtype="float32"):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=synth.DEPTH,
              hidden_dim=synth.HIDDEN, modes1=synth.MODES, modes2=synth.MODES, act_dtype=act_dtype)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m


def load_case(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    problem = str(g["problem"])
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(int(g["weight_seed"]), n_params=p, spectral_gain=float(g["spectral_gain"]))
    batch = synth.make_batch(int(g["batch_seed"]), g["preds"].shape[0], problem)
    return g, sd, batch, p


def rel(a, ref):
    return onp.rel_l2(np.asarray(a, dtype=np.float64), np.asarray(ref, dtype=np.float64))


# ------------------------------------------------------------------------------- kernel by kernel

def test_native_library_is_loaded(lib):
    from cfdbench_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH)
    from cfdbench_b200 import _lib as _l
    assert lib.fno_version() == _l.ABI_VERSION


@pytest.mark.parametrize("batch", [1, 3])
def test_dft_fwd_kernel(lib, batch):
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(0)
    x = rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)
    xd = dev(x)
    xm = torch.zeros(288, batch, 32, dtype=torch.complex64, device="cuda")  # mode-major: [k][b][c]
    _lib.check(lib.fno_spectral_dft_fwd(xd.data_ptr(), xm.data_ptr(), batch, _lib.ACT_F32, 1.0, 1.0, stream()), "dft")
    ref = onp.spectral_modes(x, 12, 12).reshape(batch, 32, 288).transpose(2, 0, 1)  # [k][b][c]
    got = xm.cpu().numpy()
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    assert err < 2e-6, err
    # scaled variant (backward uses c_ky/4096)
    _lib.check(lib.fno_spectral_dft_fwd(xd.data_ptr(), xm.data_ptr(), batch, _lib.ACT_F32, 0.25, 0.5, stream()), "dft")
    c = np.full(12, 0.5)
    c[0] = 0.25
    ref2 = (onp.spectral_modes(x, 12, 12) * c).reshape(batch, 32, 288).transpose(2, 0, 1)
    err = np.linalg.norm(xm.cpu().numpy() - ref2) / np.linalg.norm(ref2)
    assert err < 2e-6, err


def test_mode_mix_and_pack_kernels(lib):
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(1)
    batch = 200  # crosses the 128-sample tile and leaves a ragged tail
    sd = synth.make_state_dict(3, spectral_gain=100.0)
    w1, w2 = sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"]
    xm = (rng.standard_normal((288, batch, 32)) + 1j * rng.standard_normal((288, batch, 32))).astype(np.complex64)
    wk = torch.empty(288, 32, 32, dtype=torch.complex64, device="cuda")
    w1d, w2d, xmd = dev(w1), dev(w2), dev(xm)  # keep alive: the calls are asynchronous
    _lib.check(lib.fno_pack_spectral_weights(w1d.data_ptr(), w2d.data_ptr(), wk.data_ptr(), 0, stream()), "pack")
    wt = onp.stack_weights(w1, w2).reshape(32, 32, 288)  # [i][o][k]
    np.testing.assert_array_equal(wk.cpu().numpy(), wt.transpose(2, 0, 1).astype(np.complex64))
    # tensor-core operand image: per mode [hi | lo] x [n = (o, part)][kk = (i, re|im)] in K-major core matrices
    wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device="cuda")
    assert wop.numel() == 288 * 2 * 64 * 64 * 4
    _lib.check(lib.fno_pack_mix_operand(wk.data_ptr(), wop.data_ptr(), stream()), "pack operand")
    img = wop.cpu().numpy().view(np.float32).reshape(288, 2, 16, 8, 8, 4)  # [k][hi|lo][kk/4][n/8][n%8][kk%4]
    full = img.transpose(0, 1, 3, 4, 2, 5).reshape(288, 2, 64, 64).astype(np.float64)  # [k][hi|lo][n][kk]
    expand = np.empty((288, 64, 64))
    wkn = wt.transpose(2, 0, 1)  # [k][i][o]
    expand[:, 0::2, 0::2] = wkn.real.transpose(0, 2, 1)
    expand[:, 0::2, 1::2] = -wkn.imag.transpose(0, 2, 1)
    expand[:, 1::2, 0::2] = wkn.imag.transpose(0, 2, 1)
    expand[:, 1::2, 1::2] = wkn.real.transpose(0, 2, 1)
    assert np.abs(full.sum(1) - expand).max() <= 2.0 ** -21 * np.abs(expand).max()
    assert np.all((img.view(np.uint32) & 0x1FFF) == 0)  # both images are exact tf32 values
    # the one-launch pack from the parameter layout produces the same bytes, forward and adjoint
    wop2 = torch.empty_like(wop)
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wop2.data_ptr(), 0, stream()), "direct")
    assert torch.equal(wop, wop2)
    wkT0 = torch.empty(288, 32, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_pack_spectral_weights(w1d.data_ptr(), w2d.data_ptr(), wkT0.data_ptr(), 1, stream()), "packT")
    wopT, wopT2 = torch.empty_like(wop), torch.empty_like(wop)
    _lib.check(lib.fno_pack_mix_operand(wkT0.data_ptr(), wopT.data_ptr(), stream()), "pack operand T")
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wopT2.data_ptr(), 1, stream()), "direct T")
    assert torch.equal(wopT, wopT2)
    ym = torch.zeros(288, batch, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_mode_mix(xmd.data_ptr(), wop.data_ptr(), ym.data_ptr(), batch, stream()), "mix")
    ref = np.einsum("kbi,iok->kbo", xm.astype(np.complex128), wt)
    err = np.linalg.norm(ym.cpu().numpy() - ref) / np.linalg.norm(ref)
    assert err < 2e-6, err
    # small batch: one partially filled tile
    xm3 = dev(np.ascontiguousarray(xm[:, :3]))
    ym1 = torch.zeros(288, 3, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_mode_mix(xm3.data_ptr(), wop.data_ptr(), ym1.data_ptr(), 3, stream()), "mix")
    torch.cuda.synchronize()
    assert torch.equal(ym1, ym[:, :3])
    # adjoint pack + unpack
    wkT = torch.empty(288, 32, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_pack_spectral_weights(w1d.data_ptr(), w2d.data_ptr(), wkT.data_ptr(), 1, stream()), "packT")
    np.testing.assert_array_equal(wkT.cpu().numpy(), np.conj(wt).transpose(2, 1, 0).astype(np.complex64))
    g1 = torch.empty(32, 32, 12, 12, dtype=torch.complex64, device="cuda")
    g2 = torch.empty_like(g1)
    _lib.check(lib.fno_unpack_spectral_grads(wk.data_ptr(), g1.data_ptr(), g2.data_ptr(), stream()), "unpack")
    np.testing.assert_array_equal(g1.cpu().numpy(), w1)
    np.testing.assert_array_equal(g2.cpu().numpy(), w2)


@pytest.mark.parametrize("batch", [1, 3, 41])
def test_spectral_dft_fwd_bf16_planes_tensor_core_kernel(lib, batch):
    """bf16 planes through dft_fwd_tc_kernel (two chained wgmma GEMMs; the forward path of bf16 storage), which
    fno_spectral_dft_fwd runs for every bf16 plane; 41 samples = 328 plane batches, i.e. up to three per persistent CTA
    (pipeline steady state + ragged tail).
    The inputs are bf16-exact, so the comparison with the float64 oracle measures the arithmetic only."""
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(10 + batch)
    x = torch.from_numpy(rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)).to(torch.bfloat16)
    xd = x.cuda()
    xm = torch.zeros(288, batch, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_spectral_dft_fwd(xd.data_ptr(), xm.data_ptr(), batch, _lib.ACT_BF16, 1.0, 1.0, stream()), "dft tc")
    xf = x.float().numpy()
    ref = onp.spectral_modes(xf, 12, 12).reshape(batch, 32, 288).transpose(2, 0, 1)
    err = np.linalg.norm(xm.cpu().numpy() - ref) / np.linalg.norm(ref)
    assert err < 2e-6, err
    assert np.abs(xm.cpu().numpy() - ref).max() < 2e-5 * np.abs(ref).max()
    xm2 = torch.zeros_like(xm)
    _lib.check(lib.fno_spectral_dft_fwd(xd.data_ptr(), xm2.data_ptr(), batch, _lib.ACT_BF16, 0.25, 0.5, stream()), "dft tc")
    c = np.full(12, 0.5)
    c[0] = 0.25
    ref2 = (onp.spectral_modes(xf, 12, 12) * c).reshape(batch, 32, 288).transpose(2, 0, 1)
    assert np.linalg.norm(xm2.cpu().numpy() - ref2) / np.linalg.norm(ref2) < 2e-6
    xm3 = torch.zeros_like(xm)  # a second launch on the same planes: the same bits
    _lib.check(lib.fno_spectral_dft_fwd(xd.data_ptr(), xm3.data_ptr(), batch, _lib.ACT_BF16, 1.0, 1.0, stream()), "dft")
    assert np.linalg.norm(xm3.cpu().numpy() - ref) / np.linalg.norm(ref) < 2e-6
    assert torch.equal(xm3, xm)


@pytest.mark.parametrize("epi", ["gelu", "save_pre", "mul_dgelu", "plain"])
def test_block_out_kernel(lib, epi):
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(2)
    batch = 2
    ym = (rng.standard_normal((batch, 32, 24, 12)) + 1j * rng.standard_normal((batch, 32, 24, 12))) * 40.0
    x = rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)
    w0 = (rng.standard_normal((32, 32)) / 6).astype(np.float32)
    bias = rng.standard_normal(32).astype(np.float32)
    pre_in = rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)
    ymd = dev(np.ascontiguousarray(ym.reshape(batch, 32, 288).transpose(2, 0, 1)).astype(np.complex64))  # [k][b][o]
    out = torch.zeros(batch, 32, 64, 64, device="cuda")
    pre_out = torch.zeros(batch, 32, 64, 64, device="cuda")
    code = {"gelu": _lib.EPI_GELU, "save_pre": _lib.EPI_GELU_SAVE_PRE, "mul_dgelu": _lib.EPI_MUL_DGELU,
            "plain": _lib.EPI_PLAIN}[epi]
    fwd = epi in ("gelu", "save_pre")
    s0, s1 = (1 / 4096, 2 / 4096) if fwd else (1.0, 1.0)
    xd, w0td, biasd, pred = dev(x), dev(w0.T.copy()), dev(bias), dev(pre_in)  # keep alive (async launch)
    zs = torch.empty(batch, 64, 24, 32, device="cuda")
    _lib.check(lib.fno_spectral_inv_kx(ymd.data_ptr(), zs.data_ptr(), batch, s0, s1, stream()), "inv_kx")
    # K3a alone: Z[b][h][2ky+ri][o] = s_ky * sum_kx Y[b][o][kx][ky] e^{+2 pi i kx h/64}
    fh = np.exp(2j * np.pi * np.outer(np.arange(64), onp.kept_rows(64, 12)) / 64)
    zref = np.einsum("hk,bokl->bhlo", fh, ym.astype(np.complex64).astype(np.complex128)) * np.where(np.arange(12) == 0, s0, s1)[None, None, :, None]
    zgot = zs.cpu().numpy().reshape(batch, 64, 12, 2, 32)
    zgot = zgot[:, :, :, 0] + 1j * zgot[:, :, :, 1]
    assert np.linalg.norm(zgot - zref) / np.linalg.norm(zref) < 2e-6
    _lib.check(lib.fno_block_out(code, zs.data_ptr(), xd.data_ptr(), w0td.data_ptr(),
                                 biasd.data_ptr() if fwd else None, out.data_ptr(),
                                 pre_out.data_ptr() if epi == "save_pre" else None,
                                 pred.data_ptr() if epi == "mul_dgelu" else None, batch, _lib.ACT_F32,
                                 stream()), "block_out")
    ym_r = ym.astype(np.complex64).astype(np.complex128)
    spec = onp.spectral_inverse(ym_r, 64, 64, 12, 12, c0=None if fwd else 1.0, c1=None if fwd else 1.0)
    lin = spec + np.einsum("oi,bihw->bohw", w0.astype(np.float64), x.astype(np.float64))
    if fwd:
        lin = lin + bias.astype(np.float64)[None, :, None, None]
        ref = onp.gelu(lin)
    elif epi == "mul_dgelu":
        ref = lin * onp.dgelu(pre_in.astype(np.float64))
    else:
        ref = lin
    assert rel(out.cpu().numpy(), ref) < 3e-6
    if epi == "save_pre":
        assert rel(pre_out.cpu().numpy(), lin) < 3e-6


@pytest.mark.parametrize("problem", ["cavity", "cylinder"])
def test_lift_and_project_kernels(lib, problem):
    from cfdbench_b200 import _lib
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(5, n_params=p)
    batch = synth.make_batch(6, 3, problem)
    m = make_model(sd, p)
    pk = m._pack()
    a0 = torch.zeros(3, 32, 64, 64, device="cuda")
    inp_d, mk_d, cp_d = dev(batch["inputs"]), dev(batch["mask"]), dev(batch["case_params"])
    _lib.check(lib.fno_lift_fwd(inp_d.data_ptr(), mk_d.data_ptr(), cp_d.data_ptr(), C.byref(pk["struct"]),
                                a0.data_ptr(), 3, _lib.ACT_F32, stream()), "lift")
    ref = onp.conv1x1(onp.lift_features(batch["inputs"], batch["case_params"], batch["mask"]),
                      sd["fc0.weight"], sd["fc0.bias"])
    assert rel(a0.cpu().numpy(), ref) < 2e-6
    # project on a random activation
    rng = np.random.default_rng(7)
    a = rng.standard_normal((3, 32, 64, 64)).astype(np.float32)
    preds = torch.zeros(3, 2, 64, 64, device="cuda")
    a_d = dev(a)
    _lib.check(lib.fno_project_fwd(a_d.data_ptr(), mk_d.data_ptr(), C.byref(pk["struct"]),
                                   preds.data_ptr(), 3, _lib.ACT_F32, stream()), "project")
    z1 = onp.conv1x1(a.astype(np.float64), sd["fc1.weight"], sd["fc1.bias"])
    refp = onp.conv1x1(onp.gelu(z1), sd["fc2.weight"], sd["fc2.bias"]) * batch["mask"]
    assert rel(preds.cpu().numpy(), refp) < 3e-6


def test_gelu_device_accuracy(lib):
    """The erfc-polynomial GELU inside block_out: zero spectrum, identity-free path -> GELU(bias + 0)."""
    from cfdbench_b200 import _lib
    xs = np.linspace(-9, 9, 32 * 64 * 64, dtype=np.float32).reshape(1, 32, 64, 64)
    eye = np.eye(32, dtype=np.float32)
    out = torch.zeros(1, 32, 64, 64, device="cuda")
    xs_d, eye_d, zero_d = dev(xs), dev(eye), dev(np.zeros(32, np.float32))
    zs = torch.zeros(1, 64, 24, 32, device="cuda")
    _lib.check(lib.fno_block_out(_lib.EPI_GELU, zs.data_ptr(), xs_d.data_ptr(), eye_d.data_ptr(),
                                 zero_d.data_ptr(), out.data_ptr(), None, None, 1, _lib.ACT_F32, stream()), "block_out")
    ref = onp.gelu(xs.astype(np.float64))
    got = out.cpu().numpy().astype(np.float64)
    assert (np.abs(got - ref) / (1 + np.abs(ref))).max() < 6e-7  # the 1x1 runs as 3xTF32 on the tensor cores
    assert rel(got, ref) < 2e-7


# --------------------------------------------------------------------------------- whole model

@pytest.mark.parametrize("name", CASES)
def test_forward_matches_reference_golden(name):
    g, sd, batch, p = load_case(name)
    m = make_model(sd, p)
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    with torch.no_grad():
        out = m(**tb)
    assert out["preds"].is_contiguous() and out["preds"].dtype == torch.float32
    e = rel(out["preds"].cpu().numpy(), g["preds"])
    assert e < TOL, e
    for i, k in enumerate(("mse", "rmse", "mae", "nmse")):
        assert abs(out["loss"][k].item() - g["loss"][i]) < 2e-5 * abs(g["loss"][i])
    # intermediate: first block output through the C ABI pieces (act1 golden)
    nout = onp.fno_forward(sd, batch["inputs"], batch["case_params"], batch["mask"])
    assert rel(out["preds"].cpu().numpy(), nout["preds"]) < TOL


@pytest.mark.parametrize("name", CASES)
def test_rollout_matches_reference_golden(name):
    g, sd, batch, p = load_case(name)
    m = make_model(sd, p)
    steps = int(g["steps"])
    inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
    seq = m.generate_many(inp, cp, mk, steps)
    assert isinstance(seq, list) and len(seq) == steps and tuple(seq[0].shape) == tuple(inp.shape)
    gold = g["rollout"]
    # teacher-forced: step s from the golden frame s-1 (north_star: per-step output on identical inputs)
    for s in range(steps):
        prev = inp if s == 0 else torch.from_numpy(gold[s - 1]).cuda()
        with torch.no_grad():  # as reference src/test_multistep.py:108
            e = rel(m.generate(prev, cp, mk).cpu().numpy(), gold[s])
        assert e < TOL, (s, e)
    # free-running: errors compound, allow a 10x margin at the last step
    for s in range(steps):
        e = rel(seq[s].cpu().numpy(), gold[s])
        assert e < 10 * TOL, (s, e)
    # unbatched call form of test_multistep.py (reference src/test_multistep.py:102-118)
    one = m.generate_many(inp[0], cp[0], mk[0, 0], 2)
    assert tuple(one[0].shape) == (1, 2, 64, 64)
    assert rel(one[1].cpu().numpy(), gold[1][:1]) < 10 * TOL


def test_destroy_releases_library_tables_and_they_are_rebuilt(lib):
    """fno_destroy frees the constant operand tables / events the library owns on this device; the next call rebuilds them."""
    from cfdbench_b200 import _lib
    g, sd, batch, p = load_case("cavity_b2_gain200")
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items() if k != "label"}
    outs = []
    for act in ("float32", "bfloat16"):
        m = make_model(sd, p, act_dtype=act)
        m.graph_rollout = False
        with torch.no_grad():
            a = m.generate(tb["inputs"], tb["case_params"], tb["mask"])
            _lib.check(lib.fno_destroy(), "fno_destroy")
            b = m.generate(tb["inputs"], tb["case_params"], tb["mask"])
        assert torch.equal(a, b), act


def test_host_rollout_and_graph_rollout_equal_device_rollout():
    g, sd, batch, p = load_case("cylinder_b2_gain200")
    m = make_model(sd, p)
    inp, cp, mk = (torch.from_numpy(batch[k]) for k in ("inputs", "case_params", "mask"))
    m.graph_rollout = False  # every kernel launched on the stream
    dseq = m.generate_many(inp.cuda(), cp.cuda(), mk.cuda(), 4)
    hseq = m.generate_many(inp, cp, mk, 4)  # host tensors -> fno_rollout_host
    assert hseq[0].device.type == "cpu"
    for a, b in zip(dseq, hseq):
        assert torch.equal(a.cpu(), b)
    m.graph_rollout = True
    gseq = m.generate_many(inp.cuda(), cp.cuda(), mk.cuda(), 4)
    gseq2 = m.generate_many(inp.cuda(), cp.cuda(), mk.cuda(), 4)
    for a, b, c in zip(dseq, gseq, gseq2):
        assert torch.equal(a, b) and torch.equal(a, c)


# bf16 activation storage: tests/test_gpu_fused.py


def test_gradients_match_reference_golden():
    g, sd, batch, p = load_case("cylinder_b2_gain200")
    m = make_model(sd, p)
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    out = m(**tb)
    out["loss"]["nmse"].backward()
    grads = {k: v.grad.cpu().numpy() for k, v in m.named_parameters()}
    ngr = onp.fno_backward(sd, batch["inputs"], batch["case_params"], batch["mask"], batch["label"])
    for k, gv in grads.items():
        err = np.linalg.norm(gv - ngr[k]) / np.linalg.norm(ngr[k])
        assert err < 2e-5, (k, err)
    for key in g.files:
        if key.startswith("grad::"):
            k = key[6:]
            err = np.linalg.norm(grads[k] - g[key]) / np.linalg.norm(g[key])
            assert err < 5e-5, (k, err)
        elif key.startswith("gradslice::"):
            k = key[11:]
            err = np.linalg.norm(grads[k][:, :, ::4, ::4] - g[key]) / np.linalg.norm(g[key])
            assert err < 5e-5, (k, err)


def test_train_step_matches_torch_port():
    """fwd -> nmse.backward -> Adam.step x3 (reference src/train_auto.py:233-260) tracks the CPU port."""
    p = 5
    sd = synth.make_state_dict(21, n_params=p, spectral_gain=50.0)
    m = make_model(sd, p)
    pp = opt.params_from_numpy(sd, requires_grad=True)
    o_gpu = torch.optim.Adam(m.parameters(), lr=1e-3)
    o_cpu = torch.optim.Adam(list(pp.values()), lr=1e-3)
    for step in range(3):
        batch = synth.make_batch(100 + step, 4, "cavity")
        tb = {k: torch.from_numpy(v) for k, v in batch.items()}
        l_cpu = opt.train_step(pp, o_cpu, tb)
        out = m(**{k: v.cuda() for k, v in tb.items()})
        out["loss"]["nmse"].backward()
        o_gpu.step()
        o_gpu.zero_grad()
        assert abs(out["loss"]["nmse"].item() - l_cpu) < 1e-4 * abs(l_cpu), step
    for k, v in m.state_dict().items():
        a, b = v.cpu().numpy(), pp[k].detach().numpy()
        # Adam normalises the update, so tiny gradient differences can move single entries by ~lr
        assert np.linalg.norm(a - b) / np.linalg.norm(b) < 2e-3, k


# -------------------------------------------------------------- properties at BASELINE batch size

def test_full_batch_properties():
    """B=256 (BASELINE.json configs[1]): batch-permutation equivariance, determinism, and agreement of a
    few samples with the oracle (the whole batch is too slow for the float64 oracle)."""
    p = 5
    sd = synth.make_state_dict(31, n_params=p, spectral_gain=100.0)
    m = make_model(sd, p)
    batch = synth.make_batch(32, 256, "cavity", with_label=False)
    inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
    with torch.no_grad():
        y1 = m.generate(inp, cp, mk)
        y2 = m.generate(inp, cp, mk)
        assert torch.equal(y1, y2)
        perm = torch.randperm(256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
        yp = m.generate(inp[perm], cp[perm], mk[perm])
        assert torch.equal(yp, y1[perm])
    # host tensors at this size take the chunked multi-stream path (graph-replayed fno_forward per batch chunk): identical
    # result
    hseq = m.generate_many(inp.cpu(), cp.cpu(), mk.cpu(), 1)
    assert hseq[0].device.type == "cpu" and torch.equal(hseq[0], y1.cpu())
    hseq2 = m.generate_many(hseq[0], cp.cpu(), mk.cpu(), 1)  # feeding the returned (pinned) buffer back is safe
    with torch.no_grad():
        assert torch.equal(hseq2[0], m.generate(y1, cp, mk).cpu())
    idx = [0, 97, 255]
    ref = onp.fno_forward(sd, batch["inputs"][idx], batch["case_params"][idx], batch["mask"][idx])["preds"]
    assert rel(y1[idx].cpu().numpy(), ref) < TOL
    # masked pixels are exactly zero for the cylinder mask
    b2 = synth.make_batch(33, 64, "cylinder", with_label=False)
    m2 = make_model(synth.make_state_dict(34, n_params=8), 8)
    with torch.no_grad():
        y = m2.generate(*(torch.from_numpy(b2[k]).cuda() for k in ("inputs", "case_params", "mask")))
    assert float((y.cpu() * (1 - torch.from_numpy(b2["mask"]))).abs().max()) == 0.0


def test_multistep_metrics_match_reference_definition():
    """SURVEY.md 8f.1: per-step mean over cases of get_metrics(preds_u*mask, label_u*mask)
    (reference src/test_multistep.py:73-83,153-177), one launch + one D2H here."""
    from cfdbench_b200.metrics import multistep_metrics
    rng = np.random.default_rng(5)
    s_, b_ = 5, 7
    preds = rng.standard_normal((s_, b_, 2, 64, 64)).astype(np.float32)
    label = rng.standard_normal((s_, b_, 64, 64)).astype(np.float32)
    mask = (rng.random((s_, b_, 64, 64)) > 0.1).astype(np.float32)
    got = multistep_metrics(torch.from_numpy(preds).cuda(), torch.from_numpy(label).cuda(), torch.from_numpy(mask).cuda())
    assert len(got) == s_
    for s in range(s_):
        per_case = []
        for b in range(b_):
            p = preds[s, b, 0].astype(np.float64) * mask[s, b]
            l = label[s, b].astype(np.float64) * mask[s, b]
            mse = np.mean((p - l) ** 2)
            per_case.append(dict(mse=mse, nmse=mse / np.mean(l ** 2), mae=np.mean(np.abs(p - l))))
        for k in ("mse", "nmse", "mae"):
            ref = np.mean([d[k] for d in per_case])
            assert abs(got[s][k] - ref) < 2e-6 * abs(ref), (s, k, got[s][k], ref)
    # also accepts the list generate_many returns
    got2 = multistep_metrics([torch.from_numpy(preds[i]).cuda() for i in range(s_)], torch.from_numpy(label).cuda(),
                             torch.from_numpy(mask).cuda())
    assert got2 == got
