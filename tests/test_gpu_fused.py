"""GPU parity of the fused Fourier-block output stage (bf16 activation storage): `fno_mode_mix_image` +
`fno_block_fused` through the C ABI against the float64 oracle, and the whole bf16-storage model against the
bf16-boundary oracle (torch port rounding the same tensors to bf16; reference src/models/fno/fno2d.py:59-112).

Tolerances in bf16 storage mode.  Both sides round the same five hidden tensors (a_0 .. a_4) to bf16, but their
arithmetic differs in the last bits (3xTF32 tensor-core sums vs FFT + oneDNN, ~2e-7 relative), so a value that lies that
close to a bf16 rounding boundary lands on the other side (a "flip": the element moves by one bf16 ulp, |v|/128..|v|/256)
and the flip is then amplified by the layers behind it.  Two *oracles* that differ only in arithmetic precision show the
same effect: the torch port (fp32 arithmetic, the reference's library calls) and the numpy oracle (float64 arithmetic), both
rounding a_0..a_4 to bf16, are 2e-4 .. 1.6e-3 apart on the golden cases.  1e-5 therefore cannot hold between ANY two
implementations of the bf16-storage network, and the model-level tests are self-calibrating: the GPU result must be as
close to each bf16-boundary oracle as the two oracles are to each other (x2 margin).  Where flips cannot compound the
tests are strict: the fused kernel's output must be within ONE bf16 ulp (+ the fp32 evaluation error of the
pre-activation) of the correctly rounded float64 result, and only a fraction of a percent of the elements may differ at all.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import error_bounds as eb
from oracle import fno_numpy as onp
from oracle import fno_torch_port as opt

from test_gpu_parity import dev, load_case, make_model, rel, stream

pytestmark = pytest.mark.gpu


def flip_floor_and_errors(got, sd, batch):
    """(floor, e_torch, e_numpy): distance between the two bf16-boundary oracles, and of `got` to each."""
    pp = opt.params_from_numpy(sd)
    cb = {k: torch.from_numpy(np.asarray(v)) for k, v in batch.items()}
    with torch.no_grad():
        r_t = opt.forward(pp, cb["inputs"], cb["case_params"], cb["mask"], round_fn=opt.bf16_round)["preds"].numpy()
    r_n = onp.fno_forward(sd, batch["inputs"], batch["case_params"], batch["mask"], round_fn=onp.bf16_round)["preds"]
    return rel(r_t, r_n), rel(got, r_t), rel(got, r_n)


def assert_within_flip_ambiguity(got, sd, batch, what=""):
    floor, e_t, e_n = flip_floor_and_errors(got, sd, batch)
    bound = 2.0 * floor + 2e-5
    assert e_t < bound and e_n < bound, (what, "floor", floor, "vs torch16", e_t, "vs numpy16", e_n)
    return floor, e_t, e_n



@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def round_tf32(x):
    u = (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return u.view(np.float32)


def _rows():
    """row index of (kxi, ri) inside a ky block: 24 (kxi & 1) + 2 (kxi >> 1) + ri"""
    kxi = np.arange(24)
    return (24 * (kxi & 1) + 2 * (kxi >> 1))[:, None] + np.arange(2)[None, :]  # [kxi][ri]


def encode_ym_image(ym):
    """ym [B][32 o][24 kxi][12 ky] complex -> uint8 image [B][147456] as mode_mix_tc_kernel writes it."""
    b = ym.shape[0]
    vals = np.zeros((b, 12, 48, 32), np.float32)  # [b][ky][row][o]
    rows = _rows()
    y = np.asarray(ym, dtype=np.complex64)
    vals[:, :, rows[:, 0], :] = y.real.transpose(0, 3, 2, 1)
    vals[:, :, rows[:, 1], :] = y.imag.transpose(0, 3, 2, 1)
    hi = round_tf32(vals)
    lo = round_tf32(vals - hi)
    o = np.arange(32)
    img = np.zeros((b, 2, 12, 48, 32), np.float32)
    for row in range(48):
        pos = ((o // 8) ^ (row & 3)) * 8 + (o % 8)
        img[:, 0, :, row, :][..., pos] = hi[:, :, row, :]   # basic-index view first: keeps the axis order
        img[:, 1, :, row, :][..., pos] = lo[:, :, row, :]
    return img.reshape(b, -1).view(np.uint8)


def decode_ym_image(raw, b):
    """inverse of the above -> (hi + lo) as complex [B][32][24][12], plus the raw hi / lo float arrays."""
    img = np.ascontiguousarray(raw).view(np.float32).reshape(b, 2, 12, 48, 32)
    o = np.arange(32)
    val = np.zeros((b, 2, 12, 48, 32), np.float32)
    for row in range(48):
        pos = ((o // 8) ^ (row & 3)) * 8 + (o % 8)
        val[:, :, :, row, :] = img[:, :, :, row, :][..., pos]
    tot = val[:, 0].astype(np.float64) + val[:, 1].astype(np.float64)  # [b][ky][row][o]
    rows = _rows()
    y = tot[:, :, rows[:, 0], :] + 1j * tot[:, :, rows[:, 1], :]  # [b][ky][kxi][o]
    return y.transpose(0, 3, 2, 1), img


def bf16_ulp(x):
    """spacing of bf16 numbers at |x| (normal range)"""
    e = np.floor(np.log2(np.maximum(np.abs(x), 1e-30)))
    return 2.0 ** (e - 7)


def test_mode_mix_image_kernel(lib):
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(11)
    batch = 200  # crosses the 128-sample tile, ragged tail
    sd = synth.make_state_dict(3, spectral_gain=100.0)
    w1, w2 = sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"]
    xm = (rng.standard_normal((288, batch, 32)) + 1j * rng.standard_normal((288, batch, 32))).astype(np.complex64)
    w1d, w2d, xmd = dev(w1), dev(w2), dev(xm)
    wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wop.data_ptr(), 0, stream()), "pack")
    assert lib.fno_ym_image_bytes(batch) == batch * 147456
    img = torch.zeros(lib.fno_ym_image_bytes(batch), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_mode_mix_image(xmd.data_ptr(), wop.data_ptr(), img.data_ptr(), batch, stream()), "mix image")
    got, raw = decode_ym_image(img.cpu().numpy(), batch)
    wt = onp.stack_weights(w1, w2).reshape(32, 32, 288)
    ref = np.einsum("kbi,iok->bok", xm.astype(np.complex128), wt).reshape(batch, 32, 24, 12)
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    assert err < 2e-6, err
    assert np.all((raw.view(np.uint32) & 0x1FFF) == 0)  # hi and lo are exact tf32 values
    # same numbers as the mode-major kernel output, split exactly: hi + lo == fp32 result up to 2^-22
    ym = torch.zeros(288, batch, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_mode_mix(xmd.data_ptr(), wop.data_ptr(), ym.data_ptr(), batch, stream()), "mix")
    plain = ym.cpu().numpy().transpose(1, 2, 0).reshape(batch, 32, 24, 12)
    assert np.abs(got - plain).max() <= 2.0 ** -21 * np.abs(plain).max()


def test_mode_mix_ring_recycling_large_batch(lib):
    """700 samples = 6 sample tiles per mode, 12 or 18 tiles per CTA: the 4-slot A ring is reused three or more times, the B
    ring's two slots hold the CTA's first two modes and are refilled for a third (ragged last tile).
    Both outputs (mode-major ym, per-sample operand image) against float64 on a sample of modes."""
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(12)
    batch = 700
    sd = synth.make_state_dict(5, spectral_gain=100.0)
    w1, w2 = sd["blocks.1.conv0.weights1"], sd["blocks.1.conv0.weights2"]
    xm = (rng.standard_normal((288, batch, 32)) + 1j * rng.standard_normal((288, batch, 32))).astype(np.complex64)
    w1d, w2d, xmd = dev(w1), dev(w2), dev(xm)
    wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wop.data_ptr(), 0, stream()), "pack")
    ym = torch.zeros(288, batch, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_mode_mix(xmd.data_ptr(), wop.data_ptr(), ym.data_ptr(), batch, stream()), "mix")
    wt = onp.stack_weights(w1, w2).reshape(32, 32, 288)
    modes = [0, 1, 131, 132, 133, 147, 200, 286, 287]   # first / second / third round of the 132 CTAs, last modes
    ref = np.einsum("kbi,iok->kbo", xm[modes].astype(np.complex128), wt[:, :, modes])
    got = ym.cpu().numpy()
    assert np.linalg.norm(got[modes] - ref) / np.linalg.norm(ref) < 2e-6
    img = torch.zeros(lib.fno_ym_image_bytes(batch), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_mode_mix_image(xmd.data_ptr(), wop.data_ptr(), img.data_ptr(), batch, stream()), "mix image")
    dec, _ = decode_ym_image(img.cpu().numpy(), batch)
    plain = got.transpose(1, 2, 0).reshape(batch, 32, 24, 12)
    assert np.abs(dec - plain).max() <= 2.0 ** -21 * np.abs(plain).max()


@pytest.mark.parametrize("batch", [1, 3, 80])
def test_block_fused_kernel(lib, batch):
    """irfft2 (both stages on tensor cores, Z kept on chip) + 1x1 conv + bias + GELU, bf16 in / bf16 out.
    80 samples = 320 work units on 132 CTAs: every CTA runs two or three units (image ring phase wrap-around).
    Every store is checked by the bf16 interval rule; the share of stores that differ from the rounded float64 value
    (rounding flips) is printed.  Against the earlier "one ulp + 2e-6 max(1, |lin|)" rule it is stricter for large
    outputs (a store off by one ulp must have its float64 value within the bound of the rounding boundary) and looser for
    outputs near 0, where the absolute part of the bound (~1e-4 at this test's C2R scale) spans several bf16 ulps."""
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(20 + batch)
    ym = (rng.standard_normal((batch, 32, 24, 12)) + 1j * rng.standard_normal((batch, 32, 24, 12))) * 40.0
    ym = ym.astype(np.complex64)
    x = torch.from_numpy(rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)).to(torch.bfloat16)
    w0 = (rng.standard_normal((32, 32)) / 6).astype(np.float32)
    bias = rng.standard_normal(32).astype(np.float32)
    img = torch.from_numpy(encode_ym_image(ym)).cuda()
    xd, w0td, biasd = x.cuda(), dev(w0.T.copy()), dev(bias)
    out = torch.zeros(batch, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.fno_block_fused(img.data_ptr(), xd.data_ptr(), w0td.data_ptr(), biasd.data_ptr(), out.data_ptr(), batch,
                                   stream()), "block_fused")
    torch.cuda.synchronize()
    got = out.float().cpu().numpy().astype(np.float64)
    # float64 block on the mode image the kernel read (hi + lo); each store must be the bf16 rounding of a value within the
    # kernel's fp32 evaluation error (oracle/error_bounds.py: KAPPA_BLOCK_FUSED, GELU)
    dec, _ = decode_ym_image(img.cpu().numpy(), batch)
    ref, bound, _, _ = eb.block_out(dec, x.float().numpy().astype(np.float64), w0, bias, "gelu", eb.KAPPA_BLOCK_FUSED)
    assert rel(got, ref) < 3e-3, rel(got, ref)          # bf16 output rounding alone is ~1.6e-3
    flips = eb.check(f"block_fused B={batch}", got, ref, bound, tiles=eb.pixel_tiles(), bf16=True)
    print(f"\n[block_fused B={batch}] flipped share {flips:.3g}")


def test_block_fused_equals_unfused_path(lib):
    """Same block through inv_kx + block_tc (bf16 storage) and through the fused kernel: equal up to rounding flips."""
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(5)
    batch = 5
    ym = ((rng.standard_normal((batch, 32, 24, 12)) + 1j * rng.standard_normal((batch, 32, 24, 12))) * 40.0).astype(np.complex64)
    x = torch.from_numpy(rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)).to(torch.bfloat16).cuda()
    w0td, biasd = dev((rng.standard_normal((32, 32)) / 6).astype(np.float32)), dev(rng.standard_normal(32).astype(np.float32))
    ymd = dev(np.ascontiguousarray(ym.reshape(batch, 32, 288).transpose(2, 0, 1)))
    zs = torch.empty(batch, 64, 24, 32, device="cuda")
    out_a = torch.zeros(batch, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
    out_b = torch.zeros_like(out_a)
    _lib.check(lib.fno_spectral_inv_kx(ymd.data_ptr(), zs.data_ptr(), batch, 1 / 4096, 2 / 4096, stream()), "inv_kx")
    _lib.check(lib.fno_block_out(_lib.EPI_GELU, zs.data_ptr(), x.data_ptr(), w0td.data_ptr(), biasd.data_ptr(),
                                 out_a.data_ptr(), None, None, batch, _lib.ACT_BF16, stream()), "block_out")
    img = torch.from_numpy(encode_ym_image(ym)).cuda()
    _lib.check(lib.fno_block_fused(img.data_ptr(), x.data_ptr(), w0td.data_ptr(), biasd.data_ptr(), out_b.data_ptr(), batch,
                                   stream()), "block_fused")
    a, b = out_a.float().cpu().numpy().astype(np.float64), out_b.float().cpu().numpy().astype(np.float64)
    assert (a != b).mean() < 5e-3
    assert np.all(np.abs(a - b) <= 1.0001 * bf16_ulp(a) + 2e-5)


@pytest.mark.parametrize("batch,problem", [(1, "cavity"), (5, "cylinder"), (40, "cavity")])
def test_project_ws_kernel_bf16(lib, batch, problem):
    """fc1 + GELU + fc2 + mask on bf16 activations (project_tc_kernel<bf16>: wgmma with W1 as tf32 hi / lo): the inputs
    are bf16-exact, so the comparison with the float64 oracle measures the arithmetic only.
    40 samples = 2560 tiles > 132 CTAs x 4 pipelines: every pipeline runs several tiles."""
    from cfdbench_b200 import _lib
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(5, n_params=p)
    m = make_model(sd, p, act_dtype="bfloat16")
    pk = m._pack()
    rng = np.random.default_rng(7 + batch)
    a = torch.from_numpy(rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)).to(torch.bfloat16)
    mk = synth.make_batch(6, batch, problem, with_label=False)["mask"]
    a_d, mk_d = a.cuda(), dev(mk)
    preds = torch.zeros(batch, 2, 64, 64, device="cuda")
    _lib.check(lib.fno_project_fwd(a_d.data_ptr(), mk_d.data_ptr(), C.byref(pk["struct"]), preds.data_ptr(), batch,
                                   _lib.ACT_BF16, stream()), "project")
    z1 = onp.conv1x1(a.float().numpy().astype(np.float64), sd["fc1.weight"], sd["fc1.bias"])
    ref = onp.conv1x1(onp.gelu(z1), sd["fc2.weight"], sd["fc2.bias"]) * mk
    assert rel(preds.cpu().numpy(), ref) < 3e-6
    assert float(np.abs(preds.cpu().numpy() * (1 - mk)).max()) == 0.0


# ------------------------------------------------------------------------------ whole model, bf16 storage

def _bf16_oracle_forward(sd, batch):
    pp = opt.params_from_numpy(sd)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    with torch.no_grad():
        return opt.forward(pp, tb["inputs"], tb["case_params"], tb["mask"], round_fn=opt.bf16_round)["preds"].numpy()


@pytest.mark.parametrize("name", ["cavity_b2_gain200", "cylinder_b2_gain200"])
def test_bf16_forward_fused_vs_bf16_boundary_oracle(name):
    g, sd, batch, p = load_case(name)
    m = make_model(sd, p, act_dtype="bfloat16")
    assert m.fused_block
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    with torch.no_grad():
        out = m(**tb)
    got = out["preds"].cpu().numpy()
    floor, e_t, e_n = assert_within_flip_ambiguity(got, sd, batch, name)
    assert rel(got, g["preds"]) < 1e-2        # vs the fp32 reference: the cost of bf16 storage itself (2e-3 .. 6e-3)
    # the unfused bf16 path (inv_kx + block_tc) gives the same answer up to flips
    m2 = make_model(sd, p, act_dtype="bfloat16")
    m2.fused_block = False
    with torch.no_grad():
        got2 = m2(**tb)["preds"].cpu().numpy()
    assert rel(got, got2) < 2.0 * floor + 2e-5
    # masked pixels are exactly zero
    assert float(np.abs(got * (1 - batch["mask"])).max()) == 0.0
    # loss dict agrees with the oracle's loss on the same preds
    lo = onp.mse_loss(got.astype(np.float64), (batch["label"] * batch["mask"]).astype(np.float64))
    for k in ("mse", "nmse"):
        assert abs(out["loss"][k].item() - float(lo[k])) < 1e-4 * abs(float(lo[k]))


def test_bf16_rollout_20_steps_teacher_forced():
    """north_star's per-step comparison in the benched (bf16) mode: step s of the GPU from the oracle's frame s-1."""
    g, sd, batch, p = load_case("cavity_b2_gain200")
    m = make_model(sd, p, act_dtype="bfloat16")
    pp = opt.params_from_numpy(sd)
    inp, cp, mk = (torch.from_numpy(batch[k]) for k in ("inputs", "case_params", "mask"))
    cur = inp
    with torch.no_grad():
        for s in range(20):
            ref = opt.forward(pp, cur, cp, mk, round_fn=opt.bf16_round)["preds"]
            got = m.generate(cur.cuda(), cp.cuda(), mk.cuda()).cpu()
            if s % 5 == 0:   # the float64 oracle is slow: calibrate the flip floor on every fifth step
                floor = assert_within_flip_ambiguity(got.numpy(), sd, dict(inputs=cur.numpy(), case_params=batch["case_params"],
                                                                            mask=batch["mask"]), f"step {s}")[0]
            assert rel(got.numpy(), ref.numpy()) < 2.0 * floor + 2e-5, s
            cur = ref
    # free-running rollout through the graph-replayed native loop: same frames as step-by-step generate()
    seq = m.generate_many(inp.cuda(), cp.cuda(), mk.cuda(), 6)
    cur = inp.cuda()
    with torch.no_grad():
        for s in range(6):
            cur = m.generate(cur, cp.cuda(), mk.cuda())
            assert torch.equal(cur, seq[s]), s
    hseq = m.generate_many(inp, cp, mk, 6)  # host tensors
    for a, b in zip(seq, hseq):
        assert torch.equal(a.cpu(), b)


def test_bf16_full_batch_samples_and_properties():
    """BASELINE configs[1] size (B=256, bf16): three samples against the bf16-boundary oracle, determinism,
    batch-permutation equivariance."""
    p = 5
    sd = synth.make_state_dict(31, n_params=p, spectral_gain=100.0)
    m = make_model(sd, p, act_dtype="bfloat16")
    batch = synth.make_batch(32, 256, "cavity", with_label=False)
    inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
    with torch.no_grad():
        y1 = m.generate(inp, cp, mk)
        assert torch.equal(y1, m.generate(inp, cp, mk))
        perm = torch.randperm(256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
        assert torch.equal(m.generate(inp[perm], cp[perm], mk[perm]), y1[perm])
    idx = [0, 97, 255]
    sub = {k: batch[k][idx] for k in ("inputs", "case_params", "mask")}
    assert_within_flip_ambiguity(y1[idx].cpu().numpy(), sd, sub, "B=256 samples")


@pytest.mark.parametrize("act", ["bfloat16", "float32"])
def test_batch_invariance_ragged_large_batch(act):
    """A sample's prediction must not depend on the batch it travels in: 333 samples (every persistent kernel recycles its
    rings several times; ragged 128-sample mode tiles; an incomplete last round of block units, not split) against the same
    samples run as batches of 5 and of 1 -- bitwise, every kernel being free of cross-sample reductions."""
    p = 5
    sd = synth.make_state_dict(41, n_params=p, spectral_gain=100.0)
    m = make_model(sd, p, act_dtype=act)
    batch = synth.make_batch(42, 333, "cavity", with_label=False)
    inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
    with torch.no_grad():
        big = m.generate(inp, cp, mk)
        idx = torch.tensor([0, 127, 128, 255, 332], device="cuda")
        small = m.generate(inp[idx], cp[idx], mk[idx])
        one = m.generate(inp[332:333], cp[332:333], mk[332:333])
    assert torch.isfinite(big).all()
    assert torch.equal(big[idx], small)
    assert torch.equal(big[332:333], one)


def test_bf16_gradients_and_train_step_vs_port_with_rounding():
    """Training in bf16 storage (saved activations bf16, project_bwd / chan_outer bf16 templates): gradients against the
    torch port that rounds the same tensors (straight-through rounding, as the kernels do)."""
    g, sd, batch, p = load_case("cylinder_b2_gain200")
    m = make_model(sd, p, act_dtype="bfloat16")
    tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    out = m(**tb)
    out["loss"]["nmse"].backward()
    grads = {k: v.grad.cpu().numpy() for k, v in m.named_parameters()}
    pp = opt.params_from_numpy(sd, requires_grad=True)
    cb = {k: torch.from_numpy(v) for k, v in batch.items()}
    o = opt.forward(pp, cb["inputs"], cb["case_params"], cb["mask"], label=cb["label"], round_fn=opt.bf16_round_ste)
    o["loss"]["nmse"].backward()
    assert abs(out["loss"]["nmse"].item() - o["loss"]["nmse"].item()) < 2e-3 * abs(o["loss"]["nmse"].item())
    for k, gv in grads.items():
        ref = pp[k].grad.numpy()
        err = np.linalg.norm(gv - ref) / np.linalg.norm(ref)
        assert err < 2e-2, (k, err)   # bf16-rounded saved activations: gradient noise ~ 2^-9 * sqrt(depth)


def test_inference_mode_no_grad_and_view_contract():
    """reference src/train_auto.py:86 (`torch.inference_mode()`), :106 (`preds.view(-1, 1, h, w)`) and
    src/test_multistep.py:108 (`torch.no_grad()`) on the drop-in."""
    g, sd, batch, p = load_case("cavity_b2_gain200")
    for act in ("float32", "bfloat16"):
        m = make_model(sd, p, act_dtype=act).eval()
        tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
        with torch.inference_mode():
            out = m(**tb)
            input_loss = m.loss_fn(labels=tb["label"][:, :1], preds=tb["inputs"][:, :1])
        assert set(m.loss_fn.get_score_names()) <= set(out["loss"].keys())
        for k in m.loss_fn.get_score_names():
            assert isinstance(out["loss"][k].cpu().tolist(), float) and isinstance(input_loss[k].cpu().tolist(), float)
        v = out["preds"].view(-1, 1, 64, 64)
        assert tuple(v.shape) == (2 * batch["inputs"].shape[0], 1, 64, 64)
        with torch.no_grad():
            out2 = m(**tb)
            seq = m.generate_many(tb["inputs"][0], tb["case_params"][0], tb["mask"][0, 0], 3)
        assert torch.equal(out["preds"], out2["preds"]) and not out2["preds"].requires_grad
        assert len(seq) == 3 and tuple(seq[0].shape) == (1, 2, 64, 64)
        tol = 1e-5 if act == "float32" else 1e-2
        assert rel(out["preds"].cpu().numpy(), g["preds"]) < tol
