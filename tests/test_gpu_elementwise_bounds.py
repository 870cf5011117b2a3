"""Every forward kernel through its C ABI entry point, checked ELEMENT BY ELEMENT against float64 with the bounds of
oracle/error_bounds.py (|got - ref| <= kappa_stage * scale + eps_stage; bf16 stores: the bf16 rounding of some value
within that bound), at the batches where each kernel's schedule changes.  The batch lists follow the device's SM count.
`-s` prints each case's maximum of |err| / bound (bf16 stores: the share of stores that differ from the rounded float64
value), the measured headroom of the bound.  A failure names the worst element and how the failing ones group by sample,
row and tile."""
import ctypes as C

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import error_bounds as eb
from oracle import fno_numpy as onp

from test_gpu_dft_fwd_tc import _planes
from test_gpu_fused import decode_ym_image
from test_gpu_grid import _weights_struct
from test_gpu_parity import dev, stream

pytestmark = pytest.mark.gpu

STORAGE = ["float32", "bfloat16"]


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tile_batch(case):
    """project_tc / block_tc: 64 one-row tiles per sample on min(ceil(tiles / 4), n_sm) CTAs of four pipelines"""
    n4 = 4 * _n_sm()
    exact = n4 // np.gcd(64, n4)                     # tiles = a multiple of 4 n_sm: every pipeline runs the same count
    return {"one": 1,                                # one tile per pipeline, most pipelines idle
            "first_prefetch": n4 // 64 + 1,          # the first B whose tiles exceed 4 n_sm: the next-tile prefetch runs
            "exact": exact,
            "ragged": exact + 3}[case]               # a ragged last round


def _fused_batch(case):
    """block_fused: four CTAs (row chunks) per sample slot, n_sm // 4 slots striding over the batch"""
    slots = _n_sm() // 4
    return {"one": 1,
            "first_wrap": slots + 1,                 # the first CTA that runs a second unit: its rings wrap
            "ragged": 2 * slots + slots // 2}[case]  # half the CTAs run a third unit


def _acts(b, seed, act):
    """_planes' activations (per-channel DC offset and a spread of scales); fp32 ones get full fp32 mantissas"""
    x = _planes(b, seed)
    if act == "bfloat16":
        return x.cuda(), x.float().numpy().astype(np.float64)
    xf = x.float().numpy()
    xf = (xf * (1.0 + np.random.default_rng(seed).uniform(-2.0 ** -8, 2.0 ** -8, xf.shape))).astype(np.float32)
    return dev(xf), xf.astype(np.float64)


def _host(t):
    t = t.detach().cpu()
    if t.dtype == torch.bfloat16:
        t = t.float()
    return t.to(torch.complex128).numpy() if t.is_complex() else t.double().numpy()


def _modes_gpu(xm, b):
    """mode-major [288][B][32] -> [kx][ky][B][32]"""
    return _host(xm).reshape(24, 12, b, 32)


def _modes_ref(a):
    """[B][C][kx][ky] -> [kx][ky][B][C]"""
    return np.ascontiguousarray(np.broadcast_to(a, a.shape).transpose(2, 3, 0, 1))


def _report(what, **ratios):
    print(f"\n[{what}] " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))


def _spectra(b, seed, sd, layer=0):
    """realistic mode spectra: the float64 DFT of _planes activations (xm) and its mix with spectral-gain-100 weights
    (ym), both as the complex64 the kernels read"""
    x = _planes(b, seed).float().numpy().astype(np.float64)
    xm = onp.spectral_modes(x, 12, 12).astype(np.complex64)
    wt = onp.stack_weights(sd[f"blocks.{layer}.conv0.weights1"], sd[f"blocks.{layer}.conv0.weights2"])
    ym = np.einsum("bikl,iokl->bokl", xm.astype(np.complex128), wt, optimize=True).astype(np.complex64)
    return xm, ym, wt


def _mode_major(a):
    b = a.shape[0]
    return np.ascontiguousarray(a.transpose(2, 3, 0, 1).reshape(288, b, 32))


# ------------------------------------------------------------------------------------------------ 64 x 64
@pytest.mark.parametrize("act", STORAGE)
@pytest.mark.parametrize("case", ["one", "first_prefetch", "exact", "ragged"])
def test_lift_and_project(lib, case, act):
    from cfdbench_b200 import _lib
    b, p, keep = _tile_batch(case), 8, []
    sd = synth.make_state_dict(50 + b, n_params=p, spectral_gain=100.0)
    w = _weights_struct(sd, p, 64, 64, keep)
    bt = synth.make_batch(51 + b, b, "cylinder", with_label=False)
    code = _lib.ACT_F32 if act == "float32" else _lib.ACT_BF16
    inp, mk, cp = dev(bt["inputs"]), dev(bt["mask"]), dev(bt["case_params"])
    a0 = torch.empty(b, 32, 64, 64, device="cuda", dtype=torch.float32 if act == "float32" else torch.bfloat16)
    _lib.check(lib.fno_lift_fwd(inp.data_ptr(), mk.data_ptr(), cp.data_ptr(), C.byref(w), a0.data_ptr(), b, code,
                                stream()), "lift")
    feats = onp.lift_features(bt["inputs"], bt["case_params"], bt["mask"])
    ref, bound = eb.lift(feats, sd["fc0.weight"], sd["fc0.bias"], p)
    r_lift = eb.check(f"lift {act} B={b}", _host(a0), ref, bound, tiles=eb.pixel_tiles(), bf16=act == "bfloat16")
    a_d, a = _acts(b, 52 + b, act)
    preds = torch.empty(b, 2, 64, 64, device="cuda")
    _lib.check(lib.fno_project_fwd(a_d.data_ptr(), mk.data_ptr(), C.byref(w), preds.data_ptr(), b, code, stream()),
               "project")
    storage = "f32" if act == "float32" else "bf16"
    ref, bound = eb.project(a, sd["fc1.weight"], sd["fc1.bias"], sd["fc2.weight"], sd["fc2.bias"], bt["mask"],
                            eb.KAPPA_FC1[storage], 8 if act == "float32" else 5)
    r_proj = eb.check(f"project {act} B={b}", _host(preds), ref, bound, tiles=eb.pixel_tiles())
    _report(f"lift+project {act} B={b} ({case})", lift=r_lift, project=r_proj)


# bf16: test_dft_fwd_tc_every_unit's unit / tail cases; fp32 (one CTA per four planes, no persistent schedule): one
# sample, an odd batch and the largest
DFT_CASES = [("bfloat16", b) for b in (1, 2, 33, 67, 255, 256, 257)] + [("float32", b) for b in (1, 33, 257)]


@pytest.mark.parametrize("act,b", DFT_CASES)
def test_forward_dft(lib, b, act):
    from cfdbench_b200 import _lib
    x_d, x = _acts(b, 60 + b, act)
    xm = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
    code = _lib.ACT_F32 if act == "float32" else _lib.ACT_BF16
    _lib.check(lib.fno_spectral_dft_fwd(x_d.data_ptr(), xm.data_ptr(), b, code, 0.25, 0.5, stream()), "dft")
    kappa = eb.kappa_dft_f32() if act == "float32" else eb.KAPPA_DFT_BF16
    ref, bound = eb.dft(x, kappa, s0=0.25, s1=0.5)
    r = eb.check(f"dft {act} B={b}", _modes_gpu(xm, b), _modes_ref(ref), _modes_ref(bound), axes=eb.MODE_AXES,
                 tiles=eb.mode_tiles())
    _report(f"dft {act} B={b}", dft=r)


@pytest.mark.parametrize("b", [127, 128, 129])   # the 128-sample tile: one short, exact, one sample over
def test_mode_mix_all_modes(lib, b):
    from cfdbench_b200 import _lib
    sd = synth.make_state_dict(70 + b, spectral_gain=100.0)
    xm, _, wt = _spectra(b, 71 + b, sd)
    w1d, w2d = dev(sd["blocks.0.conv0.weights1"]), dev(sd["blocks.0.conv0.weights2"])
    wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wop.data_ptr(), 0, stream()), "pack")
    xmd = dev(_mode_major(xm))
    ym = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_mode_mix(xmd.data_ptr(), wop.data_ptr(), ym.data_ptr(), b, stream()), "mix")
    ref, bound = eb.mode_mix(xm.astype(np.complex128), wt)
    r = eb.check(f"mode_mix B={b}", _modes_gpu(ym, b), _modes_ref(ref), _modes_ref(bound), axes=eb.MODE_AXES,
                 tiles=eb.mode_tiles())
    img = torch.empty(lib.fno_ym_image_bytes(b), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_mode_mix_image(xmd.data_ptr(), wop.data_ptr(), img.data_ptr(), b, stream()), "mix image")
    dec, _ = decode_ym_image(img.cpu().numpy(), b)
    r_img = eb.check(f"mode_mix_image B={b}", _modes_ref(dec), _modes_ref(ref), _modes_ref(bound / eb.KAPPA_MIX
                                                                                          * eb.KAPPA_MIX_IMAGE),
                     axes=eb.MODE_AXES, tiles=eb.mode_tiles())
    _report(f"mode_mix B={b}", mode_mix=r, mode_mix_image=r_img)


@pytest.mark.parametrize("case", ["one", "first_wrap", "ragged"])
def test_mode_mix_image_and_block_fused(lib, case):
    from cfdbench_b200 import _lib
    b = _fused_batch(case)
    sd = synth.make_state_dict(80 + b, spectral_gain=100.0)
    xm, _, wt = _spectra(b, 81 + b, sd)
    w1d, w2d = dev(sd["blocks.0.conv0.weights1"]), dev(sd["blocks.0.conv0.weights2"])
    wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wop.data_ptr(), 0, stream()), "pack")
    xmd = dev(_mode_major(xm))
    img = torch.empty(lib.fno_ym_image_bytes(b), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_mode_mix_image(xmd.data_ptr(), wop.data_ptr(), img.data_ptr(), b, stream()), "mix image")
    ymix, mbound = eb.mode_mix(xm.astype(np.complex128), wt, eb.KAPPA_MIX_IMAGE)
    dec, _ = decode_ym_image(img.cpu().numpy(), b)
    r_img = eb.check(f"mode_mix_image B={b}", _modes_ref(dec), _modes_ref(ymix), _modes_ref(mbound), axes=eb.MODE_AXES,
                     tiles=eb.mode_tiles())
    x_d, x = _acts(b, 82 + b, "bfloat16")
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    bias = sd["blocks.0.w0.bias"]
    w0td, biasd = dev(np.ascontiguousarray(w0.T)), dev(bias)
    out = torch.empty(b, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.fno_block_fused(img.data_ptr(), x_d.data_ptr(), w0td.data_ptr(), biasd.data_ptr(), out.data_ptr(), b,
                                   stream()), "block_fused")
    ref, bound, _, _ = eb.block_out(dec, x, w0, bias, "gelu", eb.KAPPA_BLOCK_FUSED)   # given the image it read
    flips = eb.check(f"block_fused B={b}", _host(out), ref, bound, tiles=eb.pixel_tiles(), bf16=True)
    _report(f"block_fused B={b} ({case})", mode_mix_image=r_img, block_fused_flip_share=flips)


@pytest.mark.parametrize("act", STORAGE)
@pytest.mark.parametrize("case", ["one", "first_prefetch", "exact", "ragged"])
def test_inv_kx_and_block_out(lib, case, act):
    from cfdbench_b200 import _lib
    b = _tile_batch(case)
    sd = synth.make_state_dict(90 + b, spectral_gain=100.0)
    _, ym, _ = _spectra(b, 91 + b, sd)
    ymd = dev(_mode_major(ym))
    y = ym.astype(np.complex128)
    x_d, x = _acts(b, 92 + b, act)
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    bias = sd["blocks.0.w0.bias"]
    pre_in = np.random.default_rng(93 + b).standard_normal((b, 32, 64, 64)).astype(np.float32)
    w0td, biasd, pred = dev(np.ascontiguousarray(w0.T)), dev(bias), dev(pre_in)
    code = _lib.ACT_F32 if act == "float32" else _lib.ACT_BF16
    odt = torch.float32 if act == "float32" else torch.bfloat16
    ratios = {}
    for epi in ("gelu", "save_pre", "mul_dgelu", "plain"):
        fwd = epi in ("gelu", "save_pre")
        s0, s1 = (1 / 4096, 2 / 4096) if fwd else (1.0, 1.0)
        zs = torch.empty(b, 64, 24, 32, device="cuda")
        _lib.check(lib.fno_spectral_inv_kx(ymd.data_ptr(), zs.data_ptr(), b, s0, s1, stream()), "inv_kx")
        zref, zbound = eb.inv_kx(y, 64, s0, s1)
        zg = _host(zs).reshape(b, 64, 12, 2, 32)
        zg = (zg[:, :, :, 0] + 1j * zg[:, :, :, 1]).transpose(0, 3, 1, 2)           # -> [B][O][H][ky]
        ratios[f"inv_kx({s0:.3g})"] = eb.check(f"inv_kx B={b}", zg, zref, zbound, axes=("sample", "channel", "h", "ky"),
                                               tiles=eb.pixel_tiles(12))
        out = torch.empty(b, 32, 64, 64, device="cuda", dtype=odt)
        pre_out = torch.empty(b, 32, 64, 64, device="cuda")
        code_epi = {"gelu": _lib.EPI_GELU, "save_pre": _lib.EPI_GELU_SAVE_PRE, "mul_dgelu": _lib.EPI_MUL_DGELU,
                    "plain": _lib.EPI_PLAIN}[epi]
        _lib.check(lib.fno_block_out(code_epi, zs.data_ptr(), x_d.data_ptr(), w0td.data_ptr(),
                                     biasd.data_ptr() if fwd else None, out.data_ptr(),
                                     pre_out.data_ptr() if epi == "save_pre" else None,
                                     pred.data_ptr() if epi == "mul_dgelu" else None, b, code, stream()), "block_out")
        ref, bound, lin, lin_bound = eb.block_out(y, x, w0, bias if fwd else None, epi, eb.KAPPA_BLOCK_TC, pre_in,
                                                  s0, s1)
        ratios[epi] = eb.check(f"block_out {epi} {act} B={b}", _host(out), ref, bound, tiles=eb.pixel_tiles(),
                               bf16=act == "bfloat16")
        if epi == "save_pre":
            ratios["pre"] = eb.check(f"block_out pre {act} B={b}", _host(pre_out), lin, lin_bound,
                                     tiles=eb.pixel_tiles())
    _report(f"inv_kx+block_out {act} B={b} ({case})", **ratios)


# ------------------------------------------------------------------------------------------------ grid path
# odd H*W (every other plane only 4-byte aligned), both orientations, a tile-multiple plane (24 x 128 = 24 tiles of 128)
GRIDS = [(25, 127), (127, 25), (24, 128), (128, 24), (33, 97)]


@pytest.mark.parametrize("b", [1, 3, 70])
@pytest.mark.parametrize("gh,gw", GRIDS)
def test_grid_kernels(lib, gh, gw, b):
    from cfdbench_b200 import _lib
    rng, keep, p = np.random.default_rng(gh * 1000 + gw + b), [], 8
    sd = synth.make_state_dict(gh + gw + b, n_params=p, spectral_gain=100.0)
    w = _weights_struct(sd, p, gh, gw, keep)
    s = stream()
    inp = rng.standard_normal((b, 2, gh, gw)).astype(np.float32)
    cp = rng.standard_normal((b, p)).astype(np.float32)
    mk = (rng.random((b, gh, gw)) > 0.2).astype(np.float32)
    inp_d, cp_d, mk_d = dev(inp), dev(cp), dev(mk)
    ratios = {}
    # lift
    a0 = torch.empty(b, 32, gh, gw, device="cuda")
    _lib.check(lib.fno_grid_lift_fwd(inp_d.data_ptr(), mk_d.data_ptr(), cp_d.data_ptr(), C.byref(w), a0.data_ptr(), b,
                                     gh, gw, s), "lift")
    ref, bound = eb.lift(onp.lift_features(inp, cp, mk), sd["fc0.weight"], sd["fc0.bias"], p)
    ratios["lift"] = eb.check(f"grid lift {gh}x{gw} B={b}", _host(a0), ref, bound, tiles=eb.pixel_tiles(gw))
    # activations with a per-channel DC offset and a spread of scales
    x = rng.standard_normal((b, 32, gh, gw)) * (2.0 ** (np.arange(32) % 5 - 2))[None, :, None, None] \
        + np.arange(32)[None, :, None, None] / 8
    x = x.astype(np.float32)
    x_d, x64 = dev(x), x.astype(np.float64)
    # forward DFT
    xm = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
    _lib.check(lib.fno_grid_spectral_dft_fwd(x_d.data_ptr(), xm.data_ptr(), b, gh, gw, 0.5, 2.0, s), "dft")
    ref, bound = eb.dft(x64, eb.kappa_dft_f32(gh, gw), s0=0.5, s1=2.0)
    ratios["dft"] = eb.check(f"grid dft {gh}x{gw} B={b}", _modes_gpu(xm, b), _modes_ref(ref), _modes_ref(bound),
                             axes=eb.MODE_AXES, tiles=eb.mode_tiles())
    # inverse kx + block_out, four epilogues
    y = onp.spectral_modes(x64, 12, 12) * 0.05
    ym = y.astype(np.complex64)
    y = ym.astype(np.complex128)
    ymd = dev(_mode_major(ym))
    inv = 1.0 / (gh * gw)
    z = torch.empty(b, gh, 24, 32, device="cuda")
    _lib.check(lib.fno_grid_spectral_inv_kx(ymd.data_ptr(), z.data_ptr(), b, gh, gw, inv, 2 * inv, s), "inv_kx")
    zref, zbound = eb.inv_kx(y, gh, inv, 2 * inv)
    zg = _host(z).reshape(b, gh, 12, 2, 32)
    zg = (zg[:, :, :, 0] + 1j * zg[:, :, :, 1]).transpose(0, 3, 1, 2)
    ratios["inv_kx"] = eb.check(f"grid inv_kx {gh}x{gw} B={b}", zg, zref, zbound, axes=("sample", "channel", "h", "ky"),
                                tiles=eb.pixel_tiles(12))
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    bias = sd["blocks.0.w0.bias"]
    pre_in = rng.standard_normal((b, 32, gh, gw)).astype(np.float32)
    w0td, biasd, pred = dev(np.ascontiguousarray(w0.T)), dev(bias), dev(pre_in)
    for epi in ("gelu", "save_pre", "mul_dgelu", "plain"):
        code = {"gelu": _lib.EPI_GELU, "save_pre": _lib.EPI_GELU_SAVE_PRE, "mul_dgelu": _lib.EPI_MUL_DGELU,
                "plain": _lib.EPI_PLAIN}[epi]
        use_bias = epi in ("gelu", "save_pre")
        out = torch.empty(b, 32, gh, gw, device="cuda")
        pre = torch.empty(b, 32, gh, gw, device="cuda")
        _lib.check(lib.fno_grid_block_out(code, z.data_ptr(), x_d.data_ptr(), w0td.data_ptr(),
                                          biasd.data_ptr() if use_bias else None, out.data_ptr(), pre.data_ptr(),
                                          pred.data_ptr(), b, gh, gw, s), "block_out")
        ref, bound, lin, lin_bound = eb.block_out(y, x64, w0, bias if use_bias else None, epi, eb.KAPPA_GRID_BLOCK_OUT,
                                                  pre_in, inv, 2 * inv)
        ratios[epi] = eb.check(f"grid block_out {epi} {gh}x{gw} B={b}", _host(out), ref, bound, tiles=eb.pixel_tiles(gw))
        if epi == "save_pre":
            ratios["pre"] = eb.check(f"grid block_out pre {gh}x{gw} B={b}", _host(pre), lin, lin_bound,
                                     tiles=eb.pixel_tiles(gw))
    # projection and its backward
    a = onp.gelu(lin).astype(np.float32)
    a_d = dev(a)
    preds = torch.empty(b, 2, gh, gw, device="cuda")
    _lib.check(lib.fno_grid_project_fwd(a_d.data_ptr(), mk_d.data_ptr(), C.byref(w), preds.data_ptr(), b, gh, gw, s),
               "project")
    a64 = a.astype(np.float64)
    ref, bound = eb.project(a64, sd["fc1.weight"], sd["fc1.bias"], sd["fc2.weight"], sd["fc2.bias"], mk,
                            eb.KAPPA_FC1["grid"], 8)
    ratios["project"] = eb.check(f"grid project {gh}x{gw} B={b}", _host(preds), ref, bound, tiles=eb.pixel_tiles(gw))
    dp = rng.standard_normal((b, 2, gh, gw)).astype(np.float32)
    dp_d = dev(dp)
    dpre = torch.empty(b, 32, gh, gw, device="cuda")
    dz1 = torch.empty(min(b, _lib.BWD_CHUNK), 128, gh, gw, device="cuda")
    part = torch.empty(lib.fno_grid_bwd_partials_bytes(gh, gw), dtype=torch.uint8, device="cuda")
    g = [torch.empty(n, device="cuda") for n in (128 * 32, 128, 2 * 128, 2)]
    _lib.check(lib.fno_grid_project_bwd(a_d.data_ptr(), dp_d.data_ptr(), mk_d.data_ptr(), pred.data_ptr(), C.byref(w),
                                        dpre.data_ptr(), dz1.data_ptr(), part.data_ptr(), *[t.data_ptr() for t in g],
                                        b, gh, gw, s), "project_bwd")
    ref, bound = eb.project_bwd(a64, dp.astype(np.float64), mk, pre_in.astype(np.float64), sd["fc1.weight"],
                                sd["fc1.bias"], sd["fc2.weight"])
    ratios["project_bwd"] = eb.check(f"grid project_bwd {gh}x{gw} B={b}", _host(dpre), ref, bound,
                                     tiles=eb.pixel_tiles(gw))
    _report(f"grid {gh}x{gw} B={b}", **ratios)
