"""oracle/error_bounds.py on the CPU: its per-element bounds are sound (faithful numpy emulations of the kernels'
3xTF32 / bf16x3 arithmetic stay within them) and sharp (a defect confined to one row, one element, one bf16 tile or one kx
row of twiddles exceeds them, at the scales the GPU tests use: realistic spectra through the C2R part of block_out, the
per-mode DFT bound), while the suite's aggregate bars -- relative L2, "one ulp and < 0.5 % flipped" -- pass the single
element and the bf16 tile; and each magnitude map equals the dense |M| |x| of its stage."""
import numpy as np
import pytest

from oracle import error_bounds as eb
from oracle import fno_numpy as onp

from test_gpu_dft_fwd_tc import _planes

F32 = np.float32


def _tf32(x):
    """round to the nearest tf32 value (10 explicit mantissa bits), as the kernels' hi / lo split does"""
    u = (np.ascontiguousarray(x, dtype=F32).view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return u.view(F32)


def _split(x):
    hi = _tf32(x)
    return hi, _tf32(np.asarray(x, F32) - hi)


def _bf16x3(t):
    t1 = onp.bf16_round(t).astype(F32)
    t2 = onp.bf16_round(np.asarray(t, F32) - t1).astype(F32)
    return t1, t2, onp.bf16_round(np.asarray(t, F32) - t1 - t2).astype(F32)


def _dot(terms):
    """fp32 accumulation, one correctly rounded addition per term, in the given order: terms = [(a, b)] of float32
    arrays whose products are exact in fp32 (tf32 x tf32, bf16 x bf16)"""
    acc = None
    for a, b in terms:
        p = (a.astype(np.float64) * b).astype(F32)
        acc = p if acc is None else (acc + p).astype(F32)
    return acc


def _conv_3xtf32(x, w, single=None):
    """out[b][o][h][w] = sum_i w[o][i] x[b][i][h][w] as 3xTF32 (the 1x1 conv of block_out / fc1); where `single` (a
    boolean [B][O][H][W] mask) is set, single-pass TF32 instead"""
    xh, xl = _split(x)
    wh, wl = _split(w)
    terms = []
    for i in range(w.shape[1]):
        terms += [(wh[None, :, i, None, None], xh[:, i:i + 1]), (wl[None, :, i, None, None], xh[:, i:i + 1]),
                  (wh[None, :, i, None, None], xl[:, i:i + 1])]
    out = _dot(terms)
    if single is not None:
        one = _dot(terms[0::3])
        out = np.where(single, one, out)
    return out


def _activations(b, seed, bf16=False):
    """_planes' activations (per-channel DC offset and scale); fp32 ones get full fp32 mantissas"""
    x = _planes(b, seed).float().numpy()
    if not bf16:
        x = (x * (1.0 + np.random.default_rng(seed).uniform(-2.0 ** -8, 2.0 ** -8, x.shape))).astype(F32)
    return x


def _rel(a, ref):
    return float(np.linalg.norm(a - ref) / np.linalg.norm(ref))


# ------------------------------------------------------------------------------------------ 1x1 conv (block_out)
@pytest.fixture(scope="module")
def conv_case():
    rng = np.random.default_rng(3)
    x = _activations(2, 5)
    w0 = (rng.standard_normal((32, 32)) / 6).astype(F32)
    bias = rng.standard_normal(32).astype(F32)
    ym = _spectrum(x)
    ref, bound, _, _ = eb.block_out(ym, x.astype(np.float64), w0, bias, "plain", eb.KAPPA_BLOCK_TC)
    spec = onp.spectral_inverse(ym, 64, 64, 12, 12)     # the C2R part taken as exact: only the conv is emulated
    return x, w0, bias, ref - spec, bound


def _spectrum(x):
    """the block's spectrum as the GPU tests build it: the modes of x mixed with spectral-gain-100 weights"""
    from cfdbench_b200 import synth
    sd = synth.make_state_dict(3, spectral_gain=100.0)
    wt = onp.stack_weights(sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"])
    return np.einsum("bikl,iokl->bokl", onp.spectral_modes(x.astype(np.float64), 12, 12), wt, optimize=True)


def _add_bias(out, bias):
    return (out + bias[None, :, None, None]).astype(F32)


def test_conv_3xtf32_emulation_within_bound(conv_case):
    x, w0, bias, ref, bound = conv_case
    got = _add_bias(_conv_3xtf32(x, w0), bias)
    r = eb.check("conv 3xTF32", got, ref, bound)
    print(f"\n[conv 3xTF32 emulation] max |err|/bound {r:.3g}")
    assert r < 0.1      # the bound sits well above correct arithmetic ...


@pytest.mark.parametrize("defect", ["row", "element"])
def test_conv_single_pass_defect_exceeds_bound(conv_case, defect):
    """... and below one single-pass row or element (sample 1, row 17; element (1, 5, 17, 40))"""
    x, w0, bias, ref, bound = conv_case
    single = np.zeros(ref.shape, bool)
    if defect == "row":
        single[1, :, 17, :] = True
    else:
        single[1, 5, 17, 40] = True
    got = _add_bias(_conv_3xtf32(x, w0, single), bias)
    with pytest.raises(AssertionError, match="sample=1.*h=17"):
        eb.check(f"conv, single-pass {defect}", got, ref, bound, tiles=eb.pixel_tiles())
    agg = _rel(got, ref)
    print(f"\n[conv single-pass {defect}] rel L2 {agg:.3g}, max |err|/bound {float((np.abs(got - ref) / bound).max()):.3g}")
    if defect == "element":
        assert agg < 3e-6          # test_block_out_kernel's bar passes it


# ------------------------------------------------------------------------------------------ fc1 and the projection
@pytest.mark.parametrize("storage", ["f32", "bf16"])
def test_projection_emulation_within_bound(storage):
    from cfdbench_b200 import synth
    sd = synth.make_state_dict(5, n_params=5)
    a = _activations(1, 9)
    w1, b1 = sd["fc1.weight"].reshape(128, 32), sd["fc1.bias"]
    if storage == "f32":
        z1 = _conv_3xtf32(a, w1)
    else:   # bf16 activations are exact in tf32: two passes against W1 hi / lo
        wh, wl = _split(w1)
        z1 = _dot([t for i in range(32) for t in ((wh[None, :, i, None, None], a[:, i:i + 1]),
                                                 (wl[None, :, i, None, None], a[:, i:i + 1]))])
    z1 = _add_bias(z1, b1)
    s1 = onp.conv1x1(np.abs(a), np.abs(w1), np.abs(b1))
    r1 = eb.check("fc1", z1, onp.conv1x1(a, w1, b1), eb.KAPPA_FC1[storage] * s1)
    h = onp.gelu(z1.astype(np.float64)).astype(F32)
    w2 = sd["fc2.weight"].reshape(2, 128).astype(F32)
    out = _dot([(w2[None, :, j, None, None], h[:, j:j + 1]) for j in range(128)])
    out = _add_bias(out, sd["fc2.bias"])
    mask = (np.random.default_rng(1).random((1, 64, 64)) > 0.2).astype(F32)
    ref, bound = eb.project(a, w1, b1, w2, sd["fc2.bias"], mask, eb.KAPPA_FC1[storage], 8 if storage == "f32" else 5)
    r = eb.check("projection", out * mask[:, None], ref, bound)
    print(f"\n[projection {storage} emulation] fc1 {r1:.3g}, preds {r:.3g}")
    assert r1 < 0.1 and r < 0.1


# ------------------------------------------------------------------------------------------ bf16 forward DFT
def _dft_bf16(x, wrong_lo_kxi=None, single_pass=False):
    """dft_fwd_tc_kernel's arithmetic on bf16-exact planes x [P][64][64] -> complex [P][24 kxi][12 ky]: stage A with
    the twiddles as three bf16 terms (one fp32 accumulator per term, then added), stage B as 3xTF32 against tf32 hi / lo
    twiddles, the epilogue's two-row combination.  `wrong_lo_kxi`: that kx row uses the lo twiddles of the next row, or
    none (`single_pass`)."""
    n = np.arange(64)
    ang = 2 * np.pi * np.outer(np.arange(12), n) / 64                   # [q][w]
    parts = []
    for ta in (np.cos(ang), -np.sin(ang)):                              # G_re, G_im
        t = _bf16x3(ta)
        acc = [_dot([(x[:, :, w, None], tk[None, None, :, w]) for w in range(64)]) for tk in t]   # [P][h][q]
        parts.append(((acc[0] + acc[1]).astype(F32) + acc[2]).astype(F32))
    kx = onp.kept_rows(64, 12)
    angb = 2 * np.pi * np.outer(kx, n) / 64                             # [kxi][h]
    d = {}
    for gname, g in zip(("re", "im"), parts):
        gh, gl = _split(g)                                              # [P][h][q]
        for cname, tb in (("cos", np.cos(angb)), ("sin", np.sin(angb))):
            th, tl = _split(tb)
            if wrong_lo_kxi is not None:
                tl = tl.copy()
                tl[wrong_lo_kxi] = 0.0 if single_pass else tl[wrong_lo_kxi + 1]
            terms = []
            for h in range(64):
                terms += [(gh[:, h, None, :], th[None, :, h, None]), (gh[:, h, None, :], tl[None, :, h, None]),
                          (gl[:, h, None, :], th[None, :, h, None])]
            d[gname, cname] = _dot(terms)                               # [P][kxi][q]
    re = (d["re", "cos"] + d["im", "sin"]).astype(F32)
    im = (d["im", "cos"] - d["re", "sin"]).astype(F32)
    return re + 1j * im.astype(np.float64)


@pytest.fixture(scope="module")
def dft_case():
    x = _activations(1, 21, bf16=True)[0, :8]                                      # eight planes: one unit of the kernel
    ref, bound = eb.dft(x[None].astype(np.float64), eb.KAPPA_DFT_BF16)
    return x, ref[0], bound[0]


def test_bf16_dft_emulation_within_bound(dft_case):
    x, ref, bound = dft_case
    r = eb.check("bf16 DFT", _dft_bf16(x), ref, bound)
    print(f"\n[bf16 DFT emulation] max |err|/bound {r:.3g}")
    assert r < 0.1


@pytest.mark.parametrize("defect", ["wrong_lo", "single_pass"])
def test_bf16_dft_kx_row_defect_exceeds_bound(dft_case, defect):
    """kx = 5 with the lo twiddles of kx = 6, or single-pass (no lo twiddles at all): outside the per-mode bound, 10x
    above it where the defect is largest, while correct arithmetic stays far below it"""
    x, ref, bound = dft_case
    good = eb.check("bf16 DFT", _dft_bf16(x), ref, bound)
    got = _dft_bf16(x, wrong_lo_kxi=5, single_pass=defect == "single_pass")
    with pytest.raises(AssertionError, match="kx=5"):
        eb.check(f"bf16 DFT, {defect}", got.transpose(1, 2, 0)[..., None, :], ref.transpose(1, 2, 0)[..., None, :],
                 bound.transpose(1, 2, 0)[..., None, :], axes=eb.MODE_AXES, tiles=eb.mode_tiles())
    err = np.maximum(np.abs(got.real - ref.real), np.abs(got.imag - ref.imag)) / bound
    print(f"\n[bf16 DFT {defect} kx row] rel L2 {_rel(got, ref):.3g}, |err|/bound at kx=5 {err[:, 5].max():.3g}, "
          f"elsewhere {np.delete(err, 5, axis=1).max():.3g}")
    assert err[:, 5].max() >= 10.0 and np.delete(err, 5, axis=1).max() <= good < 0.3


# ------------------------------------------------------------------------------------------ bf16 store rule
def test_bf16_round_toward_zero_in_one_block_fused_unit():
    """B = 80 as in test_block_fused_kernel; unit (sample 3, rows 16..31, all 32 channels) stored with round-toward-zero:
    one-ulp differences on ~0.16 % of the elements, which "one ulp and < 0.5 % flipped" and the conditioned tests' old
    rule pass, and the interval rule rejects."""
    rng = np.random.default_rng(4)
    b = 80
    x = _activations(b, 4, bf16=True)
    w0 = (rng.standard_normal((32, 32)) / 6).astype(F32)
    bias = rng.standard_normal(32).astype(F32)
    ref, bound, lin, _ = eb.block_out(_spectrum(x), x.astype(np.float64), w0, bias, "gelu", eb.KAPPA_BLOCK_FUSED)
    v32 = ref.astype(F32)
    good = onp.bf16_round(v32)
    assert not eb.bf16_interval(good, ref, bound).any()
    bad = good.copy()
    rz = (v32[3, :, 16:32].view(np.uint32) & np.uint32(0xFFFF0000)).view(F32)
    bad[3, :, 16:32] = rz
    with pytest.raises(AssertionError, match="sample=3"):
        eb.check("block_fused RZ unit", bad, ref, bound, tiles=eb.pixel_tiles(), bf16=True)
    # the aggregate rules
    from test_gpu_fused import bf16_ulp
    diff = np.abs(bad - good)
    share = float((diff > 0).mean())
    assert np.all(diff <= 1.0001 * bf16_ulp(good) + 2e-6 * np.maximum(1.0, np.abs(lin))) and share < 5e-3
    print(f"\n[bf16 RZ unit] flipped share {share:.3g}")


# ------------------------------------------------------------------------------------------ magnitude maps
def _dense(fn, shape, dtype=np.float64):
    """the matrix of a linear map on arrays of `shape`, column j = fn(e_j) flattened"""
    n = int(np.prod(shape))
    cols = [np.asarray(fn(np.eye(1, n, j, dtype=dtype).reshape(shape))).ravel() for j in range(n)]
    return np.stack(cols, 1)


def test_magnitude_maps_equal_dense_abs_matrices():
    rng = np.random.default_rng(0)
    # lift / 1x1 conv: |W| |x| + |b|
    feats, w, bb = rng.standard_normal((1, 7, 3, 5)), rng.standard_normal((4, 7)), rng.standard_normal(4)
    m = _dense(lambda v: onp.conv1x1(v, w, np.zeros(4)), feats.shape)
    _, bound = eb.lift(feats, w, bb, 2)
    np.testing.assert_allclose(bound / eb.kappa_lift(2),
                               (np.abs(m) @ np.abs(feats).ravel()).reshape(1, 4, 3, 5) + np.abs(bb)[None, :, None, None])
    # forward DFT on a 24 x 26 plane: c_ky (kappa_A ||x||_2 + kappa_B ||G[:, ky]||_2), G the dense stage-A map's output
    x = rng.standard_normal((1, 1, 24, 26))
    fw = np.exp(-2j * np.pi * np.outer(np.arange(12), np.arange(26)) / 26)
    g = np.stack([fw @ x[0, 0, h] for h in range(24)])                         # [h][ky]
    want = (2.0 * np.linalg.norm(x) + 3.0 * np.linalg.norm(g, axis=0)) * eb._ky_factor(12, 0.25, 0.5)
    got = eb.dft_scale(x, (2.0, 3.0), s0=0.25, s1=0.5)
    np.testing.assert_allclose(got[0, 0], np.broadcast_to(want, (24, 12)))
    # mode mix: |.| = |Re| + |Im| of the complex weights and inputs
    xm = rng.standard_normal((2, 3, 24, 12)) + 1j * rng.standard_normal((2, 3, 24, 12))
    wt = rng.standard_normal((3, 4, 24, 12)) + 1j * rng.standard_normal((3, 4, 24, 12))
    m = _dense(lambda v: np.einsum("bikl,iokl->bokl", v, wt), xm.shape, np.complex128)
    np.testing.assert_allclose(eb.mode_mix_scale(xm, wt).ravel(), eb._cabs(m) @ eb._cabs(xm).ravel())
    # inverse kx and irfft2 (C2R): the real-linear maps on (Re Y, Im Y); each output sees Re Y_j and Im Y_j through the
    # two entries (a_j, b_j), whose modulus sqrt(a^2 + b^2) is c_ky
    ym = xm[:1, :2]
    for h, w in ((24, 24), (30, 27)):
        ref = lambda v: onp.spectral_inverse(v, h, w, 12, 12)
        a, bm = _dense(ref, ym.shape), _dense(lambda v: ref(1j * v), ym.shape)
        np.testing.assert_allclose(eb.c2r_scale(ym, h, w).ravel(), np.hypot(a, bm) @ eb._cabs(ym).ravel())
        # inverse kx is complex-linear: |Re z|, |Im z| <= sum_j |m_j| (|Re y_j| + |Im y_j|)
        m = _dense(lambda v: eb.inv_kx(v, h, 0.25, 0.5)[0], ym.shape, np.complex128)
        np.testing.assert_allclose(eb.inv_kx_scale(ym, h, 0.25, 0.5).ravel(), np.abs(m) @ eb._cabs(ym).ravel())
