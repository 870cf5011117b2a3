"""The backward stages of oracle/error_bounds.py on the CPU: numpy emulations of the kernels' arithmetic -- the 64 x 64
project backward's two 3xTF32 GEMMs (GEMM1 two-pass in bf16 storage), chan_outer's blocked fp32 sums with
reduce_partials, spectral_wgrad's per-warp complex sums -- stay well within the new bounds, and each of these defects
exceeds its bound:
  1. one 64-pixel tile of GEMM2 single-pass (dpre),       2. the same for GEMM1 (visible in dz1),
  3. one chan_outer thread tile missing one pixel group's partial,
  4. one mode of spectral_wgrad missing one warp's last sample,
  5. lift_bwd's case-parameter columns weighted with the neighbouring sample's parameters for one sample,
  6. one mode of the conjugate-transposed mix pack left unconjugated.
For each defect the test also reports whether test_gpu_train_conditioned's aggregate bar (relative L2 of each final
gradient against the float64 adjoint, backward_bar(depth = 1)) would have passed it: the defect is propagated through a
depth-1 float64 chain to every final gradient it reaches, and its largest relative L2 change is compared with the bar.
`-s` prints the table.  The new magnitude maps are checked against dense |M| |x|."""
import numpy as np
import pytest

from oracle import error_bounds as eb
from oracle import fno_numpy as onp

from test_error_bounds_host import _activations, _conv_3xtf32, _dense, _dot, _split
from test_gpu_train_conditioned import backward_bar

F32 = np.float32
BAR = backward_bar(1, "grad")


def _f32(x):
    return np.asarray(x, np.float64).astype(F32)


def _fma(a, b, c):
    """fp32 fmaf: the float64 product of two fp32 values is exact, one rounding of the sum"""
    return _f32(np.asarray(a, np.float64) * b + c)


# ------------------------------------------------------------------------------------------ a depth-1 chain
@pytest.fixture(scope="module")
def chain():
    """One cylinder sample through a depth-1 network in float64 (fp32-rounded activations): the saved tensors a_0, pre_0,
    a_1 and an upstream gradient, as the project backward and layer 0's adjoint see them."""
    from cfdbench_b200 import synth
    bt = synth.make_batch(32, 1, "cylinder", with_label=False)
    p = bt["case_params"].shape[1]
    sd = synth.make_state_dict(31, n_params=p, depth=1, spectral_gain=50.0)
    mask = bt["mask"].astype(np.float64)
    feats = onp.lift_features(bt["inputs"], bt["case_params"], mask)
    a0 = _f32(onp.conv1x1(feats, sd["fc0.weight"], sd["fc0.bias"]))
    _, pre = onp.fno_block(a0.astype(np.float64), sd, 0, return_pre=True)
    pre = _f32(pre)
    a1 = _f32(onp.gelu(pre.astype(np.float64)))
    dp = np.random.default_rng(33).standard_normal((1, 2, 64, 64)).astype(F32)
    return dict(sd=sd, feats=feats, mask=bt["mask"].reshape(1, 64, 64).astype(F32), a0=a0, pre=pre, a1=a1, dp=dp, p=p,
                params=bt["case_params"])


def _downstream(c, dpre0=None, dz1=None, ym=None):
    """Final gradients reached from layer 0's upstream gradient dpre0 (w0, weights1/2, fc0, d_inputs, d_case_params),
    from dz1 (fc1.weight, fc1.bias), or from the adjoint mix's output ym (fc0, d_inputs, d_case_params), float64."""
    sd, out = c["sd"], {}
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    if dz1 is not None:
        out["fc1.weight"] = np.einsum("bjhw,bihw->ji", dz1, c["a1"], optimize=True)
        out["fc1.bias"] = dz1.sum(axis=(0, 2, 3))
    if dpre0 is not None:
        x = c["a0"].astype(np.float64)
        out["w0.weight"] = np.einsum("bohw,bihw->oi", dpre0, x, optimize=True)
        out["w0.bias"] = dpre0.sum(axis=(0, 2, 3))
        gxs, out["weights1"], out["weights2"] = onp.spectral_conv_backward(
            x, sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"], dpre0)
        ga = gxs + np.einsum("oi,bohw->bihw", w0, dpre0, optimize=True)
    elif ym is not None:
        ga = onp.spectral_inverse(ym, 64, 64, 12, 12, c0=1.0, c1=1.0)
    else:
        return out
    out["fc0.weight"] = np.einsum("bohw,bihw->oi", ga, c["feats"], optimize=True)
    out["fc0.bias"] = ga.sum(axis=(0, 2, 3))
    wl = sd["fc0.weight"].reshape(32, -1)
    out["d_inputs"] = np.einsum("oc,bohw->bchw", wl[:, :2], ga, optimize=True)
    out["d_case_params"] = np.einsum("oj,bo->bj", wl[:, 5:], ga.sum(axis=(2, 3)), optimize=True)
    return out


def _aggregate(clean: dict, bad: dict) -> tuple:
    """largest relative L2 change of any final gradient, its name, and whether backward_bar(1) passes it"""
    rel = {k: float(np.linalg.norm(bad[k] - clean[k]) / np.linalg.norm(clean[k])) for k in clean}
    worst = max(rel, key=rel.get)
    bar = 2 * BAR if worst == "d_case_params" else BAR
    return rel[worst], worst, rel[worst] <= bar


REPORT = {}


def _report(defect, ratio, agg):
    REPORT[defect] = (ratio, agg)
    print(f"\n[{defect}] max |err|/bound {ratio:.3g}; aggregate: largest rel L2 change {agg[0]:.3g} ({agg[1]}), "
          f"backward_bar {BAR:.2g} {'PASSES it' if agg[2] else 'catches it'}")


def _max_ratio(got, ref, bound):
    if np.iscomplexobj(ref):
        err = np.maximum(np.abs(got.real - ref.real), np.abs(got.imag - ref.imag))
    else:
        err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.where(err == 0, 0.0, err / bound).max())


# ------------------------------------------------------------------------------------------ project backward (64 x 64)
def _project_bwd_tc(a, dp, mask, pre, w1, b1, w2, bf16, single1=None, single2=None):
    """project_bwd_tc_kernel's arithmetic: GEMM1 z = W1 a (3xTF32; bf16 storage: a exact, W1 hi + lo), + b1, GELU'
    (as an fp32 value), dz = (w2[0] d0 + w2[1] d1) GELU'(z), GEMM2 da = W1^T dz (3xTF32 on dz's tf32 split), times
    GELU'(pre).  single1 / single2: boolean masks of GEMM1 / GEMM2 outputs computed single-pass.  Returns (dpre, dz)."""
    if bf16:
        wh, wl = _split(w1)
        terms = [t for i in range(32) for t in ((wh[None, :, i, None, None], a[:, i:i + 1]),
                                                (wl[None, :, i, None, None], a[:, i:i + 1]))]
        z = _dot(terms)
        if single1 is not None:
            z = np.where(single1, _dot(terms[0::2]), z)
    else:
        z = _conv_3xtf32(a, w1, single1)
    z = _f32(z + b1[None, :, None, None])
    dg = _f32(onp.dgelu(z.astype(np.float64)))
    d = _f32(dp * mask[:, None])
    w2m = w2.reshape(2, 128).astype(F32)
    t = _f32(w2m[1][None, :, None, None] * d[:, 1:2].astype(np.float64))
    dz = _f32(_fma(w2m[0][None, :, None, None], d[:, 0:1], t) * dg.astype(np.float64))
    da = _conv_3xtf32(dz, np.ascontiguousarray(w1.T), single2)
    return _f32(da * onp.dgelu(pre.astype(np.float64)).astype(F32).astype(np.float64)), dz


@pytest.fixture(scope="module", params=["f32", "bf16"])
def project_case(request, chain):
    storage = request.param
    c = chain
    a = onp.bf16_round(c["a1"]).astype(F32) if storage == "bf16" else c["a1"]
    w1, b1, w2 = c["sd"]["fc1.weight"].reshape(128, 32).astype(F32), c["sd"]["fc1.bias"].astype(F32), c["sd"]["fc2.weight"]
    ref, bound, dz_ref, dz_bound = eb.project_bwd(a.astype(np.float64), c["dp"].astype(np.float64), c["mask"],
                                                  c["pre"].astype(np.float64), w1, b1, w2, eb.KAPPA_FC1[storage],
                                                  eb.KAPPA_DA["tc"], with_dz1=True)
    args = (a, c["dp"], c["mask"], c["pre"], w1, b1, w2, storage == "bf16")
    return dict(storage=storage, args=args, ref=ref, bound=bound, dz_ref=dz_ref, dz_bound=dz_bound)


def test_project_bwd_tc_emulation_within_bound(project_case):
    pc = project_case
    dpre, dz = _project_bwd_tc(*pc["args"])
    r = eb.check("dpre", dpre, pc["ref"], pc["bound"], tiles=eb.pixel_tiles())
    r_dz = eb.check("dz1", dz, pc["dz_ref"], pc["dz_bound"], tiles=eb.pixel_tiles())
    print(f"\n[project_bwd_tc {pc['storage']} emulation] dpre {r:.3g}, dz1 {r_dz:.3g}")
    assert r < 0.25 and r_dz < 0.25


@pytest.mark.parametrize("gemm", [2, 1])
def test_project_bwd_tc_single_pass_tile_exceeds_bound(project_case, chain, gemm):
    """Defects 1 and 2: the 64-pixel tile of image row 17 computed single-pass in GEMM2 (seen in dpre) or GEMM1 (dz1)"""
    pc = project_case
    single = np.zeros((1, 32 if gemm == 2 else 128, 64, 64), bool)
    single[:, :, 17, :] = True
    dpre, dz = _project_bwd_tc(*pc["args"], **({"single2": single} if gemm == 2 else {"single1": single}))
    got, ref, bound = (dpre, pc["ref"], pc["bound"]) if gemm == 2 else (dz, pc["dz_ref"], pc["dz_bound"])
    with pytest.raises(AssertionError, match="h=17"):
        eb.check(f"GEMM{gemm} single-pass tile", got, ref, bound, tiles=eb.pixel_tiles())
    dpre0, dz0 = _project_bwd_tc(*pc["args"])
    clean = _downstream(chain, dpre0.astype(np.float64), dz0.astype(np.float64))
    bad = _downstream(chain, dpre.astype(np.float64), dz.astype(np.float64))
    _report(f"{1 if gemm == 2 else 2}. GEMM{gemm} single-pass tile ({pc['storage']})",
            _max_ratio(got, ref, bound), _aggregate(clean, bad))


# ------------------------------------------------------------------------------------------ chan_outer + reduce_partials
def _reduce_partials(rows):
    """reduce_partials_kernel's order: thread row group ty adds rows ty, ty + 32, .. into four sums (four-deep while
    c + 96 < n, then round robin), adds them pairwise, then the 32 groups in order"""
    n = rows.shape[0]
    zero = np.zeros(rows.shape[1:], F32)
    red = []
    for ty in range(32):
        s = [zero] * 4
        c, u = ty, 0
        while c + 96 < n:
            s = [_f32(s[k] + rows[c + 32 * k].astype(np.float64)) for k in range(4)]
            c += 128
        while c < n:
            s[u & 3] = _f32(s[u & 3] + rows[c].astype(np.float64))
            c, u = c + 32, u + 1
        red.append(_f32(_f32(s[0] + s[1].astype(np.float64)) + _f32(s[2] + s[3].astype(np.float64)).astype(np.float64)))
    t = red[0]
    for r in red[1:]:
        t = _f32(t + r.astype(np.float64))
    return t


def _chan_outer(p, q, drop=None):
    """chan_outer_kernel<NJ, 32> + reduce_partials on P [B][NJ][4096], Q [B][32][4096] (fp32): CTA c takes items c,
    c + grid, ..; its pixel group g adds pixels g PXG .. (g + 1) PXG - 1 of each item, four per step as
    fmaf(x, ., fmaf(y, ., fmaf(z, ., fmaf(w, ., acc)))); the groups' tiles are added in order.  drop = (cta, group, tj,
    ti): that thread's tile leaves out its group's partial."""
    b, nj, ni = p.shape[0], p.shape[1], q.shape[1]
    ng, pix = 256 // nj, (64 if nj >= 128 else 128)
    pxg, chunks = pix // ng, 4096 // pix
    items = b * chunks
    grid = min(items, 296)
    acc = np.zeros((grid, ng, nj, ni), F32)
    for it0 in range(0, items, grid):
        its = np.arange(it0, min(it0 + grid, items))
        ctas, bs, p0 = its - it0, its // chunks, (its % chunks) * pix
        for g in range(ng):
            for k in [4 * qq + r for qq in range(pxg // 4) for r in (3, 2, 1, 0)]:
                px = p0 + g * pxg + k
                pv, qv = p[bs, :, px], q[bs, :, px]
                acc[ctas, g] = _fma(pv[:, :, None], qv[:, None, :], acc[ctas, g])
    if drop is not None:
        cta, g, tj, ti = drop
        rows, cols = np.arange(tj, nj, nj // 8), np.arange(ti, ni, ni // 4)
        acc[cta, g][np.ix_(rows, cols)] = 0.0
    part = acc[:, 0]
    for g in range(1, ng):
        part = _f32(part + acc[:, g].astype(np.float64))
    return _reduce_partials(part)


@pytest.mark.parametrize("b", [1, 10])   # one item per CTA; B = 10: the 296-CTA grid wraps
def test_chan_outer_emulation_and_missing_group(chain, b):
    """w0.weight = sum dpre_0 a_0^T through chan_outer<32, 32>: correct blocked sums stay within the bound; defect 3
    (one thread tile of CTA 7 without pixel group 5's partial) exceeds it at that thread's rows and columns."""
    rng = np.random.default_rng(40 + b)
    dpre = np.concatenate([_project_bwd_tc(*(chain["a1"], chain["dp"] * s, chain["mask"], chain["pre"],
                                             chain["sd"]["fc1.weight"].reshape(128, 32).astype(F32),
                                             chain["sd"]["fc1.bias"].astype(F32), chain["sd"]["fc2.weight"], False))[0]
                           for s in rng.uniform(0.1, 1.0, b)])
    a0 = np.concatenate([chain["a0"] * (1.0 + 0.1 * k) for k in range(b)]).astype(F32)
    pm, qm = dpre.reshape(b, 32, 4096), a0.reshape(b, 32, 4096)
    ref, bound = eb.Outer().add(pm.astype(np.float64), qm.astype(np.float64)).weight(eb.chain_chan_outer(b, 32))
    tiles = eb.weight_tiles(eb.chan_outer_thread(32))
    r = eb.check("chan_outer", _chan_outer(pm, qm), ref, bound, axes=eb.WEIGHT_AXES, tiles=tiles)
    got = _chan_outer(pm, qm, drop=(7, 5, 1, 2))
    with pytest.raises(AssertionError, match=r"thread tile.*\(1, 2\)"):
        eb.check("chan_outer missing group", got, ref, bound, axes=eb.WEIGHT_AXES, tiles=tiles)
    assert r < 0.25, r
    clean = {"w0.weight": _chan_outer(pm, qm).astype(np.float64)}
    _report(f"3. chan_outer thread tile missing a group (B={b}; correct sums {r:.3g})", _max_ratio(got, ref, bound),
            _aggregate(clean, {"w0.weight": got.astype(np.float64)}))


# ------------------------------------------------------------------------------------------ spectral_wgrad
def _spectral_wgrad(xm, gm, drop=None):
    """spectral_wgrad_kernel on complex64 [B][32][24][12]: warp w adds samples w, w + 4, .. as a += xr (gr, gi),
    b += xi (gr, gi) (FFMA), conj(x) g = (a.x + b.y, a.y - b.x), then the four warps in order.  drop = (kx, ky, warp):
    that mode leaves out the warp's last sample."""
    nb = xm.shape[0]
    out = None
    for w in range(4):
        z = np.zeros((32, 32, 24, 12), F32)
        ax, ay, bx, by = z, z, z, z
        samples = list(range(w, nb, 4))
        for s in samples:
            xr, xi = xm[s].real[:, None], xm[s].imag[:, None]
            gr, gi = gm[s].real[None], gm[s].imag[None]
            if drop is not None and w == drop[2] and s == samples[-1]:
                keep = np.ones((24, 12), bool)
                keep[drop[0], drop[1]] = False
                xr, xi = xr * keep, xi * keep
            ax, ay = _fma(xr, gr, ax), _fma(xr, gi, ay)
            bx, by = _fma(xi, gr, bx), _fma(xi, gi, by)
        part = _f32(ax + by.astype(np.float64)) + 1j * _f32(ay - bx.astype(np.float64)).astype(np.float64)
        out = part if out is None else (_f32(out.real + part.real) + 1j * _f32(out.imag + part.imag).astype(np.float64))
    return out


def test_spectral_wgrad_emulation_and_missing_sample(chain):
    """B = 13 (the kernel's 12-deep queue wraps): correct sums within the bound; defect 4 (mode (3, 4) without warp
    1's last sample) exceeds it at that mode only."""
    b = 13
    x = _activations(b, 41)
    xm = onp.spectral_modes(x.astype(np.float64), 12, 12).astype(np.complex64)
    g = _activations(b, 42) * np.random.default_rng(43).uniform(0.1, 1.0, (b, 1, 1, 1)).astype(F32)
    gm = (onp.spectral_modes(g.astype(np.float64), 12, 12) * eb._ky_factor(12, 1 / 4096, 2 / 4096)).astype(np.complex64)
    ref, bound = eb.spectral_wgrad(xm.astype(np.complex128), gm.astype(np.complex128), eb.chain_spectral_wgrad(b))
    axes = ("in", "out", "kx", "ky")
    tiles = {"mode (kx, ky)": lambda i, o, kx, ky: np.stack([kx, ky], 1)}
    r = eb.check("spectral_wgrad", _spectral_wgrad(xm, gm), ref, bound, axes=axes, tiles=tiles)
    got = _spectral_wgrad(xm, gm, drop=(3, 4, 1))
    with pytest.raises(AssertionError, match=r"kx=3, ky=4.*1 mode \(kx, ky\)"):
        eb.check("spectral_wgrad missing sample", got, ref, bound, axes=axes, tiles=tiles)
    assert r < 0.25, r
    clean = _spectral_wgrad(xm, gm)
    agg = _aggregate({"weights": np.concatenate([clean.real, clean.imag])},
                     {"weights": np.concatenate([got.real, got.imag])})
    _report(f"4. spectral_wgrad mode missing a warp's last sample (correct sums {r:.3g})", _max_ratio(got, ref, bound),
            agg)


# ------------------------------------------------------------------------------------------ lift_bwd, adjoint mix
def test_lift_bwd_neighbouring_params_exceeds_bound(chain):
    """Defect 5, B = 17 (lift_bwd's 16 slices take a second sample): sample 9's case-parameter columns weighted with
    sample 10's parameters."""
    b, p = 17, chain["p"]
    rng = np.random.default_rng(50)
    da0 = _f32(rng.standard_normal((b, 32, 64, 64)) * rng.uniform(0.01, 1.0, (b, 32, 1, 1)) + 0.01)
    params = rng.standard_normal((b, p))
    feats = onp.lift_features(np.repeat(chain["feats"][:, :2], b, 0), params, np.repeat(chain["mask"], b, 0))
    acc = eb.Outer().add(da0.astype(np.float64), feats)
    ref, bound = acc.weight(eb.chain_lift_bwd(b))
    bad_params = params.copy()
    bad_params[9] = params[10]
    bad = eb.Outer().add(da0.astype(np.float64),
                         onp.lift_features(np.repeat(chain["feats"][:, :2], b, 0), bad_params,
                                           np.repeat(chain["mask"], b, 0))).g
    got = _f32(bad)
    with pytest.raises(AssertionError, match=r"column=(?:[5-9]|1[0-2])\)"):
        eb.check("lift_bwd neighbouring params", got, ref, bound, axes=eb.WEIGHT_AXES)
    assert not (np.abs(_f32(ref) - ref) > bound).any()     # the fp32 rounding of the result alone stays within
    _report("5. lift_bwd case-parameter columns with the neighbour's params (B=17)", _max_ratio(got, ref, bound),
            _aggregate({"fc0.weight": ref}, {"fc0.weight": bad}))


def test_unconjugated_mode_in_adjoint_mix_exceeds_bound(chain):
    """Defect 6: the adjoint mix ym[b][i] = sum_o gm[b][o] conj(W[i][o]) with mode (5, 2) of the pack not conjugated"""
    c = chain
    sd = c["sd"]
    wt = onp.stack_weights(sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"])
    dpre0, _ = _project_bwd_tc(c["a1"], c["dp"], c["mask"], c["pre"], sd["fc1.weight"].reshape(128, 32).astype(F32),
                               sd["fc1.bias"].astype(F32), sd["fc2.weight"], False)
    gm = (onp.spectral_modes(dpre0.astype(np.float64), 12, 12) * eb._ky_factor(12, 1 / 4096, 2 / 4096))
    gm = gm.astype(np.complex64).astype(np.complex128)
    wtt = np.conj(wt).transpose(1, 0, 2, 3)
    ref, bound = eb.mode_mix(gm, wtt)
    bad_w = wtt.copy()
    bad_w[:, :, 5, 2] = wt.transpose(1, 0, 2, 3)[:, :, 5, 2]
    bad = np.einsum("bokl,oikl->bikl", gm, bad_w)
    got = bad.astype(np.complex64)
    axes = ("sample", "channel", "kx", "ky")
    with pytest.raises(AssertionError, match="kx=5, ky=2"):
        eb.check("adjoint mix, unconjugated mode", got, ref, bound, axes=axes)
    r = eb.check("adjoint mix, complex64 rounding", ref.astype(np.complex64), ref, bound, axes=axes)
    assert r < 0.1
    _report("6. adjoint mix pack with one mode unconjugated", _max_ratio(got, ref, bound),
            _aggregate(_downstream(c, ym=ref), _downstream(c, ym=bad)))


# ------------------------------------------------------------------------------------------ chains and magnitude maps
def test_chain_lengths_follow_the_launch_code():
    """the chains at the schedule changes the GPU test picks (132 SMs): chan_outer's 296-CTA cap, the project backward's
    pipelines, spectral_wgrad's warps, lift_bwd's 16 slices, reduce_partials' four-deep loop"""
    assert eb.chain_reduce_partials(32) == 1 + 33 and eb.chain_reduce_partials(296) == 10 + 33
    assert eb.chain_chan_outer(1, 32) == 16 + 7 + 34            # 32 items on 32 CTAs, 8 groups of 16 pixels
    assert eb.chain_chan_outer(10, 32) == 2 * 16 + 7 + 43       # 320 items wrap the 296 CTAs
    assert eb.chain_chan_outer(5, 128) == 2 * 32 + 1 + 43       # 320 items of 64 pixels, 2 groups of 32
    assert eb.chain_project_bwd_tc(1, 132) == 2 + 8 + 35        # 64 tiles on 64 pipelines
    assert eb.chain_project_bwd_tc(5, 132) == 2 * 2 + 8 + 42    # 320 tiles on 264 pipelines: the prefetch runs
    assert eb.chain_spectral_wgrad(13) == 2 * 4 + 4
    assert eb.chain_lift_bwd(17) == 16 * 2 + 12 + 16
    assert eb.chain_grid_chan_outer(4, 66 * 65) == 32 * 2 + 17 + 33   # 540 tiles on 528 CTAs
    assert eb.chain_grid_lift_bwd(265, 24 * 24) == 2 * (18 + 6) + 9 + 33


def test_backward_magnitude_maps_equal_dense_abs_matrices():
    rng = np.random.default_rng(7)
    # sum P Q^T: linear in P for fixed Q, |M| |P| = sum |P| |Q|; row sums sum |P|; the propagated bound |Q|^T e_P
    p, q, e = rng.standard_normal((2, 3, 5)), rng.standard_normal((2, 4, 5)), rng.random((2, 3, 5))
    m = _dense(lambda v: np.einsum("bjn,bin->ji", v, q), p.shape)
    acc = eb.Outer().add(p, q, e_p=e)
    np.testing.assert_allclose(acc.s.ravel(), np.abs(m) @ np.abs(p).ravel())
    _, bound = acc.weight(9)
    np.testing.assert_allclose(bound.ravel(), eb.kappa(9) * np.abs(m) @ np.abs(p).ravel() + np.abs(m) @ e.ravel())
    mr = _dense(lambda v: v.sum(axis=(0, 2)), p.shape)
    np.testing.assert_allclose(acc.rowsum(9)[1], eb.kappa(9) * np.abs(mr) @ np.abs(p).ravel() + mr @ e.ravel())
    # spectral_wgrad: complex-linear in G for fixed X, entries conj(x): |.| = |Re| + |Im| as for the mode mix
    xm = rng.standard_normal((3, 2, 4, 3)) + 1j * rng.standard_normal((3, 2, 4, 3))
    gm = rng.standard_normal((3, 5, 4, 3)) + 1j * rng.standard_normal((3, 5, 4, 3))
    m = _dense(lambda v: np.einsum("bikl,bokl->iokl", np.conj(xm), v), gm.shape, np.complex128)
    np.testing.assert_allclose(eb.spectral_wgrad(xm, gm, 9)[1].ravel(), eb.kappa(9) * eb._cabs(m) @ eb._cabs(gm).ravel())
    # the lift's data adjoint: d_inputs and d_case_params are linear in dL/da0
    da0, w = rng.standard_normal((2, 32, 3, 4)), rng.standard_normal((32, 8))
    chains = {"d_inputs": 4, "d_case_params": 9}
    (_, b_in), (_, b_cp) = eb.lift_data(da0, w, chains)
    for k, (fn, bnd) in enumerate(((lambda v: eb.lift_data(v, w, chains)[0][0], b_in),
                                   (lambda v: eb.lift_data(v, w, chains)[1][0], b_cp))):
        m = _dense(fn, da0.shape)
        kap = eb.kappa(chains["d_inputs" if k == 0 else "d_case_params"])
        np.testing.assert_allclose(bnd.ravel(), kap * np.abs(m) @ np.abs(da0).ravel())
