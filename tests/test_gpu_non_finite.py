"""Non-finite inputs, kernel by kernel: one element of a kernel's input -- the activation, the spectrum or a weight
operand -- set to a NaN or Inf pattern, in the last sample of the batch and on a tile edge, then

  (a) the set of non-finite output elements equals the set the float64 reference of that stage gives on the same
      poisoned input (a complex value counts as one element; only finite against non-finite is compared: 3xTF32 turns
      Inf into Inf * hi + NaN * lo, and GELU(+Inf) is NaN in the kernels, so the class of a non-finite value may differ);
  (b) every element outside that set is bit-identical to the clean run, so the kernel reads nothing outside the
      dependency cone of its output elements.

Patterns: the canonical NaN arithmetic produces (0x7fffffff / 0x7fff), the all-ones NaN (0xffffffff / 0xffff), the quiet
NaN (0x7fc00000 / 0x7fc0) and +-Inf.  The first two are what tc::round_tf32 used to turn into -0.0 / +0.0 on the
tensor-core paths.  Batches are the schedule-change batches of test_gpu_elementwise_bounds / test_gpu_backward_bounds;
the grid-generic kernels, which use no tensor cores, run the same checks on the grids there.  The footprints are taken
from the float64 references on the poisoned sample alone (every stage here computes samples independently; a clean
sample's reference is finite), except where a weight is poisoned, which reaches every sample.  The poisoned pixel is
unmasked, so the reference's (pred * mask) does not make 0 * NaN there."""
import ctypes as C

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import error_bounds as eb
from oracle import fno_numpy as onp

from test_gpu_backward_bounds import _batch_for, _run
from test_gpu_elementwise_bounds import GRIDS, _acts, _fused_batch, _mode_major, _spectra, _tile_batch
from test_gpu_fused import decode_ym_image
from test_gpu_grid import _weights_struct
from test_gpu_parity import dev, stream
from test_gpu_train_conditioned import _batch, _model, _upstream

pytestmark = pytest.mark.gpu

F32 = {"nan 0x7fffffff": 0x7fffffff, "nan 0xffffffff": 0xffffffff, "nan 0x7fc00000": 0x7fc00000,
       "+inf": 0x7f800000, "-inf": 0xff800000}
BF16 = {"nan 0x7fff": 0x7fff, "nan 0xffff": 0xffff, "nan 0x7fc0": 0x7fc0, "+inf": 0x7f80, "-inf": 0xff80}


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _value(bits, bf16):
    """the float64 value of a poison pattern (all NaNs are one NaN in the reference)"""
    u = np.array([bits << 16 if bf16 else bits], np.uint32)
    return float(u.view(np.float32)[0])


def _patterns(t):
    return BF16 if t.dtype == torch.bfloat16 else F32


def _poison(t, idx, bits):
    """a copy of t with element idx (of the float view; complex64: its real part) set to the bit pattern"""
    out = t.clone()
    f = torch.view_as_real(out) if out.is_complex() else out
    n = 8 * f.element_size()
    f.view(torch.int16 if n == 16 else torch.int32)[idx] = bits - (1 << n) if bits >> (n - 1) else bits
    return out


def _bits(t):
    t = t.detach()
    if t.is_complex():
        t = torch.view_as_real(t)
    return t.contiguous().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()]).cpu().numpy()


def _nonfinite(t):
    t = t.detach().cpu()
    if t.dtype == torch.bfloat16:
        t = t.float()
    return ~torch.isfinite(t).numpy() if not t.is_complex() else ~np.isfinite(t.numpy())


def _check(what, clean, bad, ref_nf):
    """(a) non-finite where the reference is, (b) bits of the clean run everywhere else"""
    got = _nonfinite(bad)
    assert ref_nf.shape == got.shape, (what, ref_nf.shape, got.shape)
    assert ref_nf.any(), f"{what}: the reference is finite everywhere: the set-up is wrong"
    diff = got != ref_nf
    if diff.any():
        i = tuple(int(v[0]) for v in np.nonzero(diff))
        pytest.fail(f"{what}: {int((got & ~ref_nf).sum())} elements non-finite outside the reference's footprint and "
                    f"{int((ref_nf & ~got).sum())} finite inside it (of {int(ref_nf.sum())}); first at {i}: kernel "
                    f"{'non-finite' if got[i] else 'finite'}", pytrace=False)
    keep = ~ref_nf
    cb, bb = _bits(clean), _bits(bad)
    if bad.is_complex():
        keep = np.repeat(keep[..., None], 2, -1)
    same = cb[keep] == bb[keep]
    assert same.all(), f"{what}: {int((~same).sum())} elements outside the footprint differ from the clean run"


def _edge_pixel(mask_b, w_edge=True):
    """an unmasked pixel in the last column (a tile edge) of the sample's mask, else the unmasked pixel furthest right"""
    hs, ws = np.nonzero(mask_b > 0)
    j = np.lexsort((hs, ws))[-1] if w_edge else 0
    return int(hs[j]), int(ws[j])


def _ref64(t):
    t = t.detach().cpu()
    if t.dtype == torch.bfloat16:
        t = t.float()
    return t.to(torch.complex128).numpy() if t.is_complex() else t.double().numpy()


def _modes_nf(ref):
    """non-finite set of a [B][C][kx][ky] reference in the kernels' mode-major [288][B][C] order"""
    return _mode_major(~np.isfinite(ref))


def _one_sample(nf_b, b, j):
    """a full-batch footprint that is nf_b (one sample's) at sample j, empty elsewhere (batch axis 0)"""
    out = np.zeros((b,) + nf_b.shape[1:], bool)
    out[j] = nf_b[0]
    return out


# ------------------------------------------------------------------------------------------------ 64 x 64 forward
@pytest.mark.parametrize("act", ["float32", "bfloat16"])
@pytest.mark.parametrize("case", ["first_prefetch", "ragged"])
def test_lift_and_project(lib, case, act):
    from cfdbench_b200 import _lib
    b, p, keep = _tile_batch(case), 8, []
    sd = synth.make_state_dict(50 + b, n_params=p, spectral_gain=100.0)
    w = _weights_struct(sd, p, 64, 64, keep)
    bt = synth.make_batch(51 + b, b, "cylinder", with_label=False)
    code = _lib.ACT_F32 if act == "float32" else _lib.ACT_BF16
    odt = torch.float32 if act == "float32" else torch.bfloat16
    inp, mk, cp = dev(bt["inputs"]), dev(bt["mask"]), dev(bt["case_params"])
    j = b - 1
    h, wx = _edge_pixel(bt["mask"][j, 0])

    def lift(x):
        a0 = torch.empty(b, 32, 64, 64, device="cuda", dtype=odt)
        _lib.check(lib.fno_lift_fwd(x.data_ptr(), mk.data_ptr(), cp.data_ptr(), C.byref(w), a0.data_ptr(), b, code,
                                    stream()), "lift")
        return a0

    clean = lift(inp)
    for name, bits in F32.items():
        x = _poison(inp, (j, 1, h, wx), bits)
        xb = bt["inputs"][j:j + 1].astype(np.float64)
        xb[0, 1, h, wx] = _value(bits, False)
        with np.errstate(invalid="ignore"):
            ref, _ = eb.lift(onp.lift_features(xb, bt["case_params"][j:j + 1], bt["mask"][j:j + 1]), sd["fc0.weight"],
                             sd["fc0.bias"], p)
        _check(f"lift {act} B={b} {name}", clean, lift(x), _one_sample(~np.isfinite(ref), b, j))

    a_d, a = _acts(b, 52 + b, act)

    def project(x):
        preds = torch.empty(b, 2, 64, 64, device="cuda")
        _lib.check(lib.fno_project_fwd(x.data_ptr(), mk.data_ptr(), C.byref(w), preds.data_ptr(), b, code, stream()),
                   "project")
        return preds

    clean = project(a_d)
    for name, bits in _patterns(a_d).items():
        for c in (0, 31):
            x = _poison(a_d, (j, c, h, wx), bits)
            ab = a[j:j + 1].copy()
            ab[0, c, h, wx] = _value(bits, act == "bfloat16")
            with np.errstate(invalid="ignore", over="ignore"):
                ref, _ = eb.project(ab, sd["fc1.weight"], sd["fc1.bias"], sd["fc2.weight"], sd["fc2.bias"],
                                    bt["mask"][j:j + 1], 1.0, 8)
            _check(f"project {act} B={b} channel {c} {name}", clean, project(x), _one_sample(~np.isfinite(ref), b, j))


DFT_CASES = [("bfloat16", b) for b in (1, 33, 257)] + [("float32", b) for b in (1, 33)]


@pytest.mark.parametrize("act,b", DFT_CASES)
def test_forward_dft(lib, b, act):
    from cfdbench_b200 import _lib
    x_d, x = _acts(b, 60 + b, act)
    code = _lib.ACT_F32 if act == "float32" else _lib.ACT_BF16
    j = b - 1

    def dft(t):
        xm = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
        _lib.check(lib.fno_spectral_dft_fwd(t.data_ptr(), xm.data_ptr(), b, code, 0.25, 0.5, stream()), "dft")
        return xm

    clean = dft(x_d)
    for name, bits in _patterns(x_d).items():
        for c, h, w in ((31, 63, 63), (0, 0, 0)):
            xb = x[j:j + 1].copy()
            xb[0, c, h, w] = _value(bits, act == "bfloat16")
            with np.errstate(invalid="ignore"):
                ref = onp.spectral_modes(xb, 12, 12)
            nf = np.zeros((288, b, 32), bool)
            nf[:, j:j + 1] = _modes_nf(ref)
            _check(f"dft {act} B={b} ({c}, {h}, {w}) {name}", clean, dft(_poison(x_d, (j, c, h, w), bits)), nf)


def _mix_operand(lib, w1, w2):
    from cfdbench_b200 import _lib
    w1d, w2d = dev(w1), dev(w2)   # named: a temporary's memory could be reused by the next upload before the launch
    wop = torch.empty(lib.fno_mix_operand_bytes(), dtype=torch.uint8, device="cuda")
    _lib.check(lib.fno_pack_mix_operand_from_weights(w1d.data_ptr(), w2d.data_ptr(), wop.data_ptr(), 0, stream()),
               "pack")
    return wop


@pytest.mark.parametrize("b", [127, 129])
def test_mode_mix(lib, b):
    """fno_mode_mix and fno_mode_mix_image (decoded to hi + lo), a poisoned mode of the spectrum and of weights1"""
    from cfdbench_b200 import _lib
    sd = synth.make_state_dict(70 + b, spectral_gain=100.0)
    xm, _, wt = _spectra(b, 71 + b, sd)
    w1, w2 = sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"]
    j = b - 1

    def run(xmd, wop):
        ym = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
        _lib.check(lib.fno_mode_mix(xmd.data_ptr(), wop.data_ptr(), ym.data_ptr(), b, stream()), "mix")
        img = torch.empty(lib.fno_ym_image_bytes(b), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fno_mode_mix_image(xmd.data_ptr(), wop.data_ptr(), img.data_ptr(), b, stream()), "mix image")
        dec, _ = decode_ym_image(img.cpu().numpy(), b)
        return ym, torch.from_numpy(_mode_major(dec.astype(np.complex64)))

    xmd, wop = dev(_mode_major(xm)), _mix_operand(lib, w1, w2)
    clean = run(xmd, wop)
    for name, bits in F32.items():
        v = _value(bits, False)
        for kx, ky, i in ((23, 11, 31), (0, 0, 0)):
            x64 = xm[j:j + 1].astype(np.complex128)
            x64[0, i, kx, ky] = v + 1j * x64[0, i, kx, ky].imag
            with np.errstate(invalid="ignore"):
                ref = np.einsum("bikl,iokl->bokl", x64, wt)
            nf = np.zeros((288, b, 32), bool)
            nf[:, j:j + 1] = _modes_nf(ref)
            bad = run(_poison(xmd, (12 * kx + ky, j, i, 0), bits), wop)
            _check(f"mode_mix B={b} xm ({kx}, {ky}, {i}) {name}", clean[0], bad[0], nf)
            _check(f"mode_mix_image B={b} xm ({kx}, {ky}, {i}) {name}", clean[1], bad[1], nf)
        # weights1[i][o][kx][ky], the weight operand: every sample's mode (kx, ky), channel o
        w1b = w1.copy()
        w1b.real.view(np.int32)[31, 5, 11, 11] = np.int64(bits).astype(np.uint32).view(np.int32)
        wt_b = onp.stack_weights(w1b, w2)
        with np.errstate(invalid="ignore"):
            ref = np.einsum("bikl,iokl->bokl", xm.astype(np.complex128), wt_b)
        bad = run(xmd, _mix_operand(lib, w1b, w2))
        _check(f"mode_mix B={b} weights1 {name}", clean[0], bad[0], _modes_nf(ref))
        _check(f"mode_mix_image B={b} weights1 {name}", clean[1], bad[1], _modes_nf(ref))


@pytest.mark.parametrize("case", ["first_wrap", "ragged"])
def test_block_fused(lib, case):
    """fno_block_fused from a poisoned image (the image of a poisoned spectrum) and from a poisoned activation"""
    from cfdbench_b200 import _lib
    b = _fused_batch(case)
    sd = synth.make_state_dict(80 + b, spectral_gain=100.0)
    xm, _, wt = _spectra(b, 81 + b, sd)
    wop = _mix_operand(lib, sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"])
    x_d, x = _acts(b, 82 + b, "bfloat16")
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    bias = sd["blocks.0.w0.bias"]
    w0td, biasd = dev(np.ascontiguousarray(w0.T)), dev(bias)
    j = b - 1

    def image(xmd):
        img = torch.empty(lib.fno_ym_image_bytes(b), dtype=torch.uint8, device="cuda")
        _lib.check(lib.fno_mode_mix_image(xmd.data_ptr(), wop.data_ptr(), img.data_ptr(), b, stream()), "mix image")
        return img

    def fused(img, xt):
        out = torch.empty(b, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
        _lib.check(lib.fno_block_fused(img.data_ptr(), xt.data_ptr(), w0td.data_ptr(), biasd.data_ptr(), out.data_ptr(),
                                       b, stream()), "block_fused")
        return out

    xmd = dev(_mode_major(xm))
    img0 = image(xmd)
    dec0, _ = decode_ym_image(img0.cpu().numpy(), b)
    clean = fused(img0, x_d)
    for name, bits in F32.items():
        img = image(_poison(xmd, (12 * 23 + 0, j, 7, 0), bits))
        dec, _ = decode_ym_image(img.cpu().numpy(), b)
        with np.errstate(invalid="ignore"):
            ref, _, _, _ = eb.block_out(dec[j:j + 1], x[j:j + 1], w0, bias, "gelu", 1.0)
        _check(f"block_fused B={b} image {name}", clean, fused(img, x_d), _one_sample(~np.isfinite(ref), b, j))
    for name, bits in BF16.items():
        xb = x[j:j + 1].copy()
        xb[0, 3, 63, 63] = _value(bits, True)
        with np.errstate(invalid="ignore"):
            ref, _, _, _ = eb.block_out(dec0[j:j + 1], xb, w0, bias, "gelu", 1.0)
        _check(f"block_fused B={b} x {name}", clean, fused(img0, _poison(x_d, (j, 3, 63, 63), bits)),
               _one_sample(~np.isfinite(ref), b, j))


@pytest.mark.parametrize("act", ["float32", "bfloat16"])
@pytest.mark.parametrize("case", ["first_prefetch", "ragged"])
def test_inv_kx_and_block_out(lib, case, act):
    """fno_spectral_inv_kx from a poisoned spectrum; fno_block_out (GELU epilogue, and the pre-activation it saves)
    from a poisoned z, a poisoned activation and a poisoned W0 entry"""
    from cfdbench_b200 import _lib
    b = _tile_batch(case)
    sd = synth.make_state_dict(90 + b, spectral_gain=100.0)
    _, ym, _ = _spectra(b, 91 + b, sd)
    ymd = dev(_mode_major(ym))
    y = ym.astype(np.complex128)
    x_d, x = _acts(b, 92 + b, act)
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    bias = sd["blocks.0.w0.bias"]
    biasd = dev(bias)
    code = _lib.ACT_F32 if act == "float32" else _lib.ACT_BF16
    odt = torch.float32 if act == "float32" else torch.bfloat16
    s0, s1 = 1 / 4096, 2 / 4096
    j = b - 1

    def inv_kx(t):
        zs = torch.empty(b, 64, 24, 32, device="cuda")
        _lib.check(lib.fno_spectral_inv_kx(t.data_ptr(), zs.data_ptr(), b, s0, s1, stream()), "inv_kx")
        return zs

    def block_out(zs, xt, w0t):
        out = torch.empty(b, 32, 64, 64, device="cuda", dtype=odt)
        pre = torch.empty(b, 32, 64, 64, device="cuda")
        _lib.check(lib.fno_block_out(_lib.EPI_GELU_SAVE_PRE, zs.data_ptr(), xt.data_ptr(), w0t.data_ptr(),
                                     biasd.data_ptr(), out.data_ptr(), pre.data_ptr(), None, b, code, stream()),
                   "block_out")
        return out, pre

    def z_nf(yb, kx, ky, o):
        """The float64 inverse DFT over kx makes every h, re and im, non-finite.  Exception: the kernel runs it in real
        arithmetic on the re and im parts and never multiplies by an exact-zero twiddle, so a non-finite Re y(kx) stays
        out of Im z(h) where sin(2 pi kx h / 64) is exactly 0 and out of Re z(h) where the cosine is."""
        with np.errstate(invalid="ignore"):
            zr, _ = eb.inv_kx(yb, 64, s0, s1)                             # [1][O][H][ky]
        nf = ~np.isfinite(zr).transpose(0, 2, 3, 1)                       # -> [1][H][ky][O]
        nf = np.repeat(nf[:, :, :, None, :], 2, 3)                        # [1][H][ky][re|im][O]
        for h in range(64):
            r = (kx * h) % 64
            if r in (0, 32):
                nf[0, h, ky, 1, o] = False
            if r in (16, 48):
                nf[0, h, ky, 0, o] = False
        return nf.reshape(1, 64, 24, 32)

    w0t_d = dev(np.ascontiguousarray(w0.T))
    z0 = inv_kx(ymd)
    clean = block_out(z0, x_d, w0t_d)
    for name, bits in F32.items():
        v = _value(bits, False)
        yb = y[j:j + 1].copy()
        yb[0, 9, 23, 11] = v + 1j * yb[0, 9, 23, 11].imag
        zb = inv_kx(_poison(ymd, (12 * 23 + 11, j, 9, 0), bits))
        _check(f"inv_kx B={b} {name}", z0, zb, _one_sample(z_nf(yb, 63, 11, 9), b, j))   # kx index 23 is kx = 63
        # block_out fed the poisoned z (the C2R reads the whole h row of every ky)
        zh = _ref64(zb[j:j + 1]).reshape(1, 64, 12, 2, 32)
        zc = (zh[:, :, :, 0] + 1j * zh[:, :, :, 1]).transpose(0, 3, 1, 2)   # [1][O][H][ky]
        with np.errstate(invalid="ignore", over="ignore"):
            lin = np.fft.irfft(np.concatenate([zc * np.where(np.arange(12) == 0, s0, s1 / 2) * 4096,
                                               np.zeros((1, 32, 64, 21))], -1), 64, axis=-1) \
                + onp.conv1x1(x[j:j + 1], w0, bias)
        nf = _one_sample(~np.isfinite(lin), b, j)
        got = block_out(zb, x_d, w0t_d)
        _check(f"block_out pre {act} B={b} z {name}", clean[1], got[1], nf)
        _check(f"block_out {act} B={b} z {name}", clean[0], got[0], nf)
    for name, bits in _patterns(x_d).items():
        xb = x[j:j + 1].copy()
        xb[0, 17, 0, 63] = _value(bits, act == "bfloat16")
        with np.errstate(invalid="ignore"):
            _, _, lin, _ = eb.block_out(y[j:j + 1], xb, w0, bias, "save_pre", 1.0, s0=s0, s1=s1)
        got = block_out(z0, _poison(x_d, (j, 17, 0, 63), bits), w0t_d)
        _check(f"block_out {act} B={b} x {name}", clean[0], got[0], _one_sample(~np.isfinite(lin), b, j))
    for name, bits in F32.items():
        w0b = w0.copy()
        w0b[30, 2] = _value(bits, False)
        with np.errstate(invalid="ignore"):
            _, _, lin, _ = eb.block_out(y, x, w0b, bias, "save_pre", 1.0, s0=s0, s1=s1)
        w0t_b = _poison(w0t_d, (2, 30), bits)
        got = block_out(z0, x_d, w0t_b)
        _check(f"block_out {act} B={b} W0 {name}", clean[1], got[1], ~np.isfinite(lin))


# ------------------------------------------------------------------------------------------------ grid path (control)
@pytest.mark.parametrize("gh,gw", GRIDS)
def test_grid_kernels(lib, gh, gw):
    from cfdbench_b200 import _lib
    b, p, keep = 3, 8, []
    rng = np.random.default_rng(gh * 1000 + gw)
    sd = synth.make_state_dict(gh + gw, n_params=p, spectral_gain=100.0)
    w = _weights_struct(sd, p, gh, gw, keep)
    s = stream()
    j = b - 1
    x = (rng.standard_normal((b, 32, gh, gw)) + np.arange(32)[None, :, None, None] / 8).astype(np.float32)
    x_d, x64 = dev(x), x.astype(np.float64)
    mk = np.ones((b, gh, gw), np.float32)
    mk_d = dev(mk)
    inv = 1.0 / (gh * gw)

    def dft(t):
        xm = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
        _lib.check(lib.fno_grid_spectral_dft_fwd(t.data_ptr(), xm.data_ptr(), b, gh, gw, 0.5, 2.0, s), "dft")
        return xm

    def project(t):
        preds = torch.empty(b, 2, gh, gw, device="cuda")
        _lib.check(lib.fno_grid_project_fwd(t.data_ptr(), mk_d.data_ptr(), C.byref(w), preds.data_ptr(), b, gh, gw, s),
                   "project")
        return preds

    y = (onp.spectral_modes(x64, 12, 12) * 0.05).astype(np.complex64)
    ymd = dev(_mode_major(y))

    def inv_kx(t):
        z = torch.empty(b, gh, 24, 32, device="cuda")
        _lib.check(lib.fno_grid_spectral_inv_kx(t.data_ptr(), z.data_ptr(), b, gh, gw, inv, 2 * inv, s), "inv_kx")
        return z

    clean = dft(x_d), project(x_d), inv_kx(ymd)
    for name, bits in F32.items():
        v = _value(bits, False)
        xb = x64[j:j + 1].copy()
        xb[0, 31, gh - 1, gw - 1] = v
        xp = _poison(x_d, (j, 31, gh - 1, gw - 1), bits)
        with np.errstate(invalid="ignore", over="ignore"):
            nf = np.zeros((288, b, 32), bool)
            nf[:, j:j + 1] = _modes_nf(onp.spectral_modes(xb, 12, 12))
            _check(f"grid dft {gh}x{gw} {name}", clean[0], dft(xp), nf)
            ref, _ = eb.project(xb, sd["fc1.weight"], sd["fc1.bias"], sd["fc2.weight"], sd["fc2.bias"], mk[j:j + 1],
                                1.0, 8)
            _check(f"grid project {gh}x{gw} {name}", clean[1], project(xp), _one_sample(~np.isfinite(ref), b, j))
            yb = y[j:j + 1].astype(np.complex128)
            yb[0, 4, 12, 0] = v + 1j * yb[0, 4, 12, 0].imag
            zr, _ = eb.inv_kx(yb, gh, inv, 2 * inv)
            nfz = np.repeat((~np.isfinite(zr)).transpose(0, 2, 3, 1)[:, :, :, None, :], 2, 3).reshape(1, gh, 24, 32)
            _check(f"grid inv_kx {gh}x{gw} {name}", clean[2], inv_kx(_poison(ymd, (12 * 12 + 0, j, 4, 0), bits)),
                   _one_sample(nfz, b, j))


# ------------------------------------------------------------------------------------------------ backward
BWD = [pytest.param("cavity", "float32", _batch_for, "chunks", id="64-f32-chunks"),
       pytest.param("cavity", "bfloat16", _batch_for, "chunks", id="64-bf16-chunks"),
       pytest.param("cavity", "float32", _batch_for, "prefetch", id="64-f32-prefetch"),
       pytest.param((66, 65), "float32", None, 4, id="66x65-B4"),
       pytest.param((25, 127), "float32", None, 3, id="25x127-B3")]


@pytest.mark.parametrize("where,act,batch_of,case", BWD)
def test_backward_stages(where, act, batch_of, case):
    """one element of d(preds) poisoned (channel c of the last sample, an unmasked pixel in the last column): the
    projection's backward is non-finite at that pixel only (dpre_0, every channel); the fc2 gradients in row c only;
    from the DFT of dpre_0 on every stage of that sample (gm, ym, z, dL/da0, d_inputs, d_case_params); every other
    sample bit-identical; the fc1, W0, spectral and lift weight gradients non-finite throughout (each sums over the
    poisoned pixel or mode)."""
    b = case if batch_of is None else batch_of(case)
    p, depth = 5, 1
    seed = 9100 + b
    sd = synth.make_state_dict(seed, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(seed + 1, b, where, p)
    gh, gw = bt["inputs"].shape[-2:]
    gp = _upstream(seed + 2, (b, 2, gh, gw))
    m = _model(sd, p, depth, act)
    j, c = b - 1, 1
    h, w = _edge_pixel(bt["mask"].reshape(b, gh, gw)[j])
    clean = _run(m, bt, gp)
    names = {"dpre0": "pixel", "gm": "sample", "ym": "sample", "z": "sample", "da0": "sample", "d_in": "sample",
             "d_cp": "sample"}
    for name, bits in F32.items():
        bad_gp = gp.copy()
        bad_gp.view(np.uint32)[j, c, h, w] = bits
        with np.errstate(invalid="ignore", over="ignore"):
            ref, _ = eb.project_bwd(clean["aL"][j:j + 1], bad_gp[j:j + 1].astype(np.float64),
                                    bt["mask"].reshape(b, gh, gw)[j:j + 1].astype(np.float64), clean["pre"][j:j + 1],
                                    sd["fc1.weight"], sd["fc1.bias"], sd["fc2.weight"])
        bad = _run(m, bt, bad_gp)
        for k, scope in names.items():
            cl, bd = torch.from_numpy(clean[k]), torch.from_numpy(bad[k])
            bax = 0
            if k in ("gm", "ym"):                     # mode-major [288][B][32]
                cl, bd, bax = cl.reshape(288, b, 32), bd.reshape(288, b, 32), 1
            nf = np.zeros(cl.shape, bool)
            if scope == "pixel":
                nf[j] = ~np.isfinite(ref[0])
            else:
                idx = [slice(None)] * nf.ndim
                idx[bax] = j
                nf[tuple(idx)] = True
            _check(f"{where} {act} B={b} {k} {name}", cl, bd, nf)
        for k, g in clean["grads"].items():
            nf = np.ones(g.shape, bool)
            if k.startswith("fc2."):
                nf[:] = False
                nf[c] = True
            _check(f"{where} {act} B={b} {k} {name}", torch.from_numpy(g), torch.from_numpy(bad["grads"][k]), nf)


# ------------------------------------------------------------------------------------------------ a diverging rollout
S, K = 4, 1   # rollout steps; the 0-based step at which the rollout first turns non-finite
FLT_MAX = float(np.finfo(np.float32).max)


def _diverging(grid):
    """A seeded model that is positively homogeneous (no biases, the lift reads u and v only) with fc2 scaled by 1e31,
    so each step multiplies the field by ~1e29, and a split whose cases start from frames scaled by 1e-15: step 0's
    predictions stay below 1e15 (their squared sums finite in fp32), step 1's would reach ~1e43."""
    sd = synth.make_state_dict(11, n_params=5, spectral_gain=100.0)
    for k in sd:
        if k.endswith("bias"):
            sd[k] = np.zeros_like(sd[k])
    sd["fc0.weight"][:, 2:] = 0.0
    sd["fc2.weight"] = (sd["fc2.weight"] * np.float32(1e31)).astype(np.float32)
    feats, cps = synth.make_split(3, 3, "cavity" if grid == (64, 64) else "tube", frames=(S + 1, S + 1))
    for f in feats:
        f[0, :2] *= np.float32(1e-15)
    return sd, feats, cps


class _Split:
    """the reference dataset layout of the cases: inputs = frames[:-1], labels = frames[1:], one S-step window each"""

    def __init__(self, feats, cps):
        self.inputs = torch.from_numpy(np.concatenate([f[:-1] for f in feats]))
        self.labels = torch.from_numpy(np.concatenate([f[1:] for f in feats]))
        self.case_ids = np.concatenate([[c] * (len(f) - 1) for c, f in enumerate(feats)])
        self.time_step_size = 1
        self.case_params = [{f"p{i}": float(v) for i, v in enumerate(cp)} for cp in cps]

    def __len__(self):
        return len(self.inputs)


@pytest.mark.parametrize("grid, act", [((64, 64), "float32"), ((64, 64), "bfloat16"), ((66, 65), "float32")],
                         ids=["64-f32", "64-bf16", "66x65"])
def test_diverging_rollout_metrics(grid, act):
    """infer_multistep's and evaluate_rollout_auto's per-step metrics are finite before step K and non-finite from K on,
    where the fp32 reference rollout first overflows; its float64 twin shows that rounding cannot move K (step K - 1 is
    100x below FLT_MAX, step K would be 100x above it)."""
    from cfdbench_b200 import Fno2d, evaluate_rollout_auto, infer_multistep, loss_name_to_fn
    from oracle import fno_torch_port as tp
    sd, feats, cps = _diverging(grid)
    x = np.stack([f[0, :2] for f in feats])
    mk = np.stack([f[0, 2] for f in feats])
    cp = np.stack(cps)
    with np.errstate(invalid="ignore", over="ignore"):
        r64 = onp.rollout(sd, x, cp, mk, K + 1)
    peak = [np.abs(r).reshape(len(feats), -1).max(1) for r in r64]
    assert peak[K - 1].max() <= FLT_MAX / 100 and peak[K].min() >= 100 * FLT_MAX, peak
    with torch.no_grad():
        r32 = tp.rollout(tp.params_from_numpy(sd), torch.from_numpy(x), torch.from_numpy(cp),
                         torch.from_numpy(mk[:, None]), S)
    assert all(bool(torch.isfinite(r).all()) for r in r32[:K])
    assert all(not bool(torch.isfinite(r[i]).all()) for r in r32[K:K + 1] for i in range(len(feats)))
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act).cuda()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    got = {"infer_multistep": infer_multistep(m, feats, [torch.from_numpy(c) for c in cps], infer_steps=S),
           "evaluate_rollout_auto": evaluate_rollout_auto(m, _Split(feats, cps), S)["steps"]}
    report = {k: ["".join("f" if np.isfinite(v) else "x" for v in row.values()) for row in rows]
              for k, rows in got.items()}
    print(f"\n[diverging {grid} {act}] per-step (mse, nmse, mae) finite (f) / non-finite (x): {report}")
    for what, rows in got.items():
        assert len(rows) == S
        for s, row in enumerate(rows):
            fin = [bool(np.isfinite(v)) for v in row.values()]
            assert all(fin) if s < K else not any(fin), f"{what} step {s}: {row}"
