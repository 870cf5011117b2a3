"""TEST INFRASTRUCTURE -- per-element error bounds of every kernel stage against float64.

A relative L2 over a whole output cannot see a defect confined to one tile, one image row or one element (a ragged last
tile, the first refill after a ring wraps, an edge row): one element computed single-pass TF32 moves the relative L2 of a
1x1 conv by 1e-7 but that element by 2^-11 of its magnitude.  So each stage here returns its float64 reference `ref` and
a per-element `bound`, and a kernel output passes when, on EVERY element,

    |got - ref| <= bound = kappa_stage * scale + eps_stage,

where `scale` is the stage's linear map applied to absolute values (|W| |x| + |b| for a 1x1 conv, the sums of |Y| for the
inverse DFTs, every twiddle having modulus 1; the forward DFTs use per-mode l2 norms instead, see KAPPA_DFT_BF16) and eps_stage is the absolute error of a GELU fit where one is applied.  The
maps are the oracle's own (`fno_numpy`), applied to |.|.

kappa_stage is derived from the stage's arithmetic (the derivation of each is next to its constant below):
  * accumulation: an fp32 dot product of n additions (FFMA chains, or tensor-core accumulation, which may truncate rather
    than round, hence U = 2^-23 per addition) has |error| <= n U sum|terms| in the worst case, but that bound is sqrt(n)
    times looser than what rounding errors of varying sign add up to, and with it a defect of 2^-12 per term in a K = 64
    contraction (a wrong tf32 lo term) would stay under the bar.  So the rounding part of kappa is LAMBDA sqrt(n) U
    sum|terms|, the form of the probabilistic bound of Higham & Mary (SIAM J. Sci. Comput. 41, 2019).  Their guarantee
    alone does not make it hold on every element: in their model each element exceeds it with probability up to
    2 exp(-LAMBDA^2 / 2) = 7e-4, and a check covers 1e6 .. 1e7 elements.  What does is that the actual rounding errors
    are far smaller than the model allows: they behave like sums of independent errors whose spread is set by the
    partial sums, which cancel, not by sum|terms|.  The float64 emulations of tests/test_error_bounds_host.py stay at
    0.002 .. 0.07 of the bounds, and the largest |err| / bound over all elements measured on an H100 80GB HBM3 (SXM,
    700 W power limit) by tests/test_gpu_elementwise_bounds.py, next to each constant, is 0.38 (grid inv_kx) and
    otherwise 0.15 or less (the forward DFTs, on their own per-mode bound: up to 0.55);
  * splits, worst case: 3xTF32 (a_hi b_hi + a_hi b_lo + a_lo b_hi, round-to-nearest split, |a - a_hi - a_lo| <= 2^-22 |a|)
    drops a_lo b_lo and the two split residuals: at most 3 * 2^-22 |a||b| per product;
  * constants: three bf16 terms carry 24 significant bits, 2^-24 |t|; a float32 twiddle table 2^-24 |t|.
The kappas on sum|terms| scales are below 1.5e-5, more than 30x below the 2^-11 relative error of a single-pass TF32 product, which is what
a pass skipped on one tile looks like.

A bf16 store is checked exactly: the stored value must be the bf16 rounding of SOME value within the bound of the float64
reference (`bf16_interval`), i.e. bf16(ref - bound) <= got <= bf16(ref + bound); bf16 rounding is monotone.

`check` reports the worst element by its coordinates and how the failing elements group by sample, row and tile.
"""
from __future__ import annotations

import numpy as np

from oracle import fno_numpy as onp

U = 2.0 ** -23                   # one fp32 addition (truncation allowed)
LAMBDA = 4.0                     # confidence factor of the probabilistic accumulation bound
SPLIT_3XTF32 = 3 * 2.0 ** -22    # per product of a 3xTF32 pass
SPLIT_2XTF32 = 2.0 ** -22        # x (exact in tf32, e.g. bf16) times W_hi + W_lo: only W's residual
TWIDDLE = 2.0 ** -24             # float32 twiddle table, or a constant carried by three bf16 terms
GELU_FIT = {8: 2.7e-7, 5: 6.4e-7}   # |fit - GELU| in fp32, absolute (fno_common.cuh)
DGELU_FIT = 1e-6                 # |dgelu_erf - GELU'| in fp32, absolute: erfc fit 1.5e-8, MUFU.EX2 in the Gaussian ~2^-22
SUP_DGELU = 1.13                 # sup |GELU'| = 1.1289: an error e in GELU's argument moves GELU by at most 1.13 e
SUP_D2GELU = 0.8                 # sup |GELU''| = 2 phi(0) = 0.798


def kappa(n_add: int, split: float = 0.0) -> float:
    """rounding of n_add fp32 additions (probabilistic, see the module docstring) plus the worst-case split error"""
    return LAMBDA * np.sqrt(n_add) * U + split


# ------------------------------------------------------------------------------------------ kappa of each kernel stage
# lift (fno_lift_fwd, grid_lift_kernel): a chain of 5 + p FFMA plus the bias
def kappa_lift(p: int) -> float:
    return kappa(6 + p)      # measured 0.15 (fp32 store, 64 x 64 and grids)


# Forward DFTs.  With sum |x| as the scale (the DFT's |M| |x|, the same for every mode of a plane) a defect of 2^-12 per
# term in one kx row stays under any sound bar, so the DFT bound is per mode, in the Gaussian model of rounding: every
# product and every addition perturbs the sum by an independent zero-mean error.  Stage A (along w) of row h sums n_A
# terms whose partial sums are at most sqrt(k) ||x_h||_2 (Cauchy-Schwarz), so its rounding error has a standard deviation
# of at most u n_A / sqrt(2) ||x_h||_2 (u = 2^-24 per addition); 64 rows reach the output through twiddles of modulus 1,
# giving u n_A / sqrt(2) ||x||_2.  Stage B (along h) likewise gives u n_B / sqrt(2) ||G[:, ky]||_2, G the float64 partial
# DFT along w.  The Cauchy-Schwarz bound on the partial sums makes these deviations sqrt(n / 2) times larger than those
# of a random walk, so LAMBDA_DFT = 1.5 of them is the bar; with the representation errors (twiddles, tf32 splits) on
# the same l2 norms:  c_ky (kappa_A ||x||_2 + kappa_B ||G[:, ky]||_2).  A kx row without its lo twiddles errs by about
# 2^-12 ||G[:, ky]||_2: 13x the bound in the emulation of tests/test_error_bounds_host.py, where correct arithmetic stays at
# 0.075 of it; on the H100 the kernels reach 0.375 (bf16), 0.55 (fp32, 64 x 64) and 0.37 (grids) of it.
UR = 2.0 ** -24
LAMBDA_DFT = 1.5


def _kappa_l2(n_add: int, rep: float) -> float:
    return LAMBDA_DFT * n_add / np.sqrt(2.0) * UR + rep


# fp32 forward DFT (register FFT codelets; grid_dft_kernel): a real DFT along w (W terms), then a complex one along h
# (2 H real terms), float32 twiddles in each stage, one scale multiply
def kappa_dft_f32(h: int = 64, w: int = 64) -> tuple:
    return _kappa_l2(w, TWIDDLE), _kappa_l2(2 * h + 1, TWIDDLE)   # measured 0.55 at 64 x 64 (B = 257), 0.37 on grids


# bf16 forward DFT (dft_fwd_tc_kernel): stage A, x exact times the three bf16 terms of the twiddles, one accumulator of
# 64 per term, the three added (66 additions, 2^-24); G stored fp32 and split tf32 (3xTF32, K = 64: 192 additions,
# 3 2^-22), the epilogue adds two accumulator rows and scales (2)
KAPPA_DFT_BF16 = (_kappa_l2(66, TWIDDLE), _kappa_l2(194, SPLIT_3XTF32))   # measured 0.375 (B = 255)
# mode mix (mode_mix_tc_kernel): real-expanded K = 64, 3xTF32
KAPPA_MIX = kappa(192, SPLIT_3XTF32)                  # measured 0.10 (B = 128)
# mode_mix_image writes the fp32 result as tf32 hi + lo: their sum is within 2^-22 of it
KAPPA_MIX_IMAGE = KAPPA_MIX + 2.0 ** -22              # measured 0.11 (B = 128)
# inverse DFT along kx (inv_kx_kernel, grid_inv_kx_kernel): 24 complex terms = 48 FFMA, float32 twiddles, one scale
KAPPA_INV_KX = kappa(50, TWIDDLE)      # measured 0.026 at 64 x 64, 0.38 on the grids (127 x 25, B = 70)
# block_out (block_tc_kernel): C2R along w (E, K = 24) and the 1x1 conv (K = 32) in ONE 3xTF32 chain, bias in the
# epilogue: 3 (24 + 32) + 1 = 169 additions; plus the inv_kx error Z carries (|E| sums it with the same weights c_ky)
KAPPA_BLOCK_TC = kappa(169, SPLIT_3XTF32) + KAPPA_INV_KX   # measured 0.064 (MUL_DGELU), pre 0.055
# block_fused_kernel: GEMM1 (inverse kx, 3xTF32, K = 48: 144), Zt re-split (2^-22), GEMM2: E Zt (3xTF32, K = 24: 72)
# and x W0 (three bf16 terms of W0, K = 32: 96, 2^-24), bias: 314 additions and three split errors.  The input image
# is taken as given (its own error is KAPPA_MIX_IMAGE's).
KAPPA_BLOCK_FUSED = kappa(314, 2 * SPLIT_3XTF32 + 2.0 ** -22 + TWIDDLE)   # bf16 stores: all within, 0.07 % flipped
# grid_block_out_kernel: C2R along w (24 FFMA, float32 twiddles), conv (32 FFMA), bias, plus the carried inv_kx error
KAPPA_GRID_BLOCK_OUT = kappa(57, TWIDDLE) + KAPPA_INV_KX   # measured 0.068 (MUL_DGELU)
# fc1 of the projection: fp32 storage 3xTF32, K = 32, + bias (97); bf16 storage x exact, W1 hi + lo (65); FFMA on grids
KAPPA_FC1 = {"f32": kappa(97, SPLIT_3XTF32), "bf16": kappa(65, SPLIT_2XTF32), "grid": kappa(33)}
# fc2: 128 FFMA per output (four lane partial sums added in a fixed order) + bias
KAPPA_FC2 = kappa(129)   # projection measured 0.014 (64 x 64), 0.028 (grids); grid_project_bwd's dpre 0.068
# da = W1^T dz1 of the project backward (K = 128 hidden units).  project_bwd_tc_kernel's GEMM2 is 3xTF32 in both storage
# modes (dz1 is fp32 either way): 3 x 128 additions; its split error covers dz1's re-split into tf32 hi / lo in the
# epilogue (one of the three 2^-22 terms) and W1's.  Its GEMM1 is fc1 (KAPPA_FC1["f32"] / ["bf16"]).  grid: 128 FFMA.
KAPPA_DA = {"tc": kappa(384, SPLIT_3XTF32), "grid": kappa(128)}   # dpre measured 0.060 (64 x 64), 0.056 (grids);
# dz1 (kappa(3) and the GELU' terms of project_bwd) 0.084 (64 x 64), 0.095 (grids)


# ------------------------------------------------------------------------------------------ references and scales
def _ky_factor(m2: int, s0: float, s1: float) -> np.ndarray:
    c = np.full(m2, float(s1))
    c[0] = s0
    return c


def lift(feats: np.ndarray, w: np.ndarray, b: np.ndarray, p: int):
    """a0 = fc0(features): (ref, bound).  scale = |W| |features| + |b|."""
    ref = onp.conv1x1(feats, w, b)
    scale = onp.conv1x1(np.abs(feats), np.abs(w), np.abs(b))
    return ref, kappa_lift(p) * scale


def dft_scale(x: np.ndarray, kappa: tuple, m1: int = 12, m2: int = 12, s0: float = 1.0, s1: float = 1.0) -> np.ndarray:
    """Per-mode bound of the two-stage truncated DFT (see KAPPA_DFT_BF16): c_ky (kappa_A ||x||_2 + kappa_B ||G[:, ky]||_2)
    over each plane, G[h][ky] = sum_w x[h][w] e^{-2 pi i ky w / W}; [B][C][2 m1][m2]."""
    w = x.shape[-1]
    fw = np.exp(-2j * np.pi * np.outer(np.arange(m2), np.arange(w)) / w)
    g = np.einsum("bchw,kw->bchk", x, fw, optimize=True)
    gn = np.sqrt((np.abs(g) ** 2).sum(axis=-2))                        # [B][C][ky]
    xn = np.sqrt((np.abs(x) ** 2).sum(axis=(-2, -1)))[..., None]       # [B][C][1]
    per_ky = (kappa[0] * xn + kappa[1] * gn) * _ky_factor(m2, s0, s1)
    return np.broadcast_to(per_ky[..., None, :], x.shape[:2] + (2 * m1, m2))


def dft(x: np.ndarray, kappa: tuple, m1: int = 12, m2: int = 12, s0: float = 1.0, s1: float = 1.0):
    """Kept modes of x scaled by s0 (ky = 0) / s1: (ref, bound), complex ref [B][C][2 m1][m2], bound for Re and Im;
    kappa = (kappa_A, kappa_B) of the two stages."""
    ref = onp.spectral_modes(x, m1, m2) * _ky_factor(m2, s0, s1)
    return ref, dft_scale(x, kappa, m1, m2, s0, s1)


def _cabs(z: np.ndarray) -> np.ndarray:
    return np.abs(z.real) + np.abs(z.imag)


def mode_mix_scale(xm: np.ndarray, wt: np.ndarray) -> np.ndarray:
    """sum_i (|Re x| + |Im x|)(|Re w| + |Im w|): xm [B][I][kx][ky], wt [I][O][kx][ky] -> [B][O][kx][ky]."""
    return np.einsum("bikl,iokl->bokl", _cabs(xm), _cabs(wt), optimize=True)


def mode_mix(xm: np.ndarray, wt: np.ndarray, kappa: float = KAPPA_MIX):
    ref = np.einsum("bikl,iokl->bokl", xm, wt, optimize=True)
    return ref, kappa * mode_mix_scale(xm, wt)


def inv_kx_scale(ym: np.ndarray, h: int, s0: float, s1: float) -> np.ndarray:
    """|M| (|Re Y| + |Im Y|) of the inverse DFT along kx (twiddles of modulus 1): [B][O][H][ky], for Re and Im of Z."""
    m2 = ym.shape[-1]
    tot = _cabs(ym).sum(axis=-2) * _ky_factor(m2, s0, s1)       # [B][O][ky]
    return np.broadcast_to(tot[:, :, None, :], ym.shape[:2] + (h, m2))


def inv_kx(ym: np.ndarray, h: int, s0: float, s1: float, kappa: float = KAPPA_INV_KX):
    """Z[b][o][h][ky] = s_ky sum_kx Y e^{+2 pi i kx h / H} over the kept rows: (ref complex, bound)."""
    m1 = ym.shape[-2] // 2
    fh = np.exp(2j * np.pi * np.outer(np.arange(h), onp.kept_rows(h, m1)) / h)
    ref = np.einsum("hk,bokl->bohl", fh, ym, optimize=True) * _ky_factor(ym.shape[-1], s0, s1)
    return ref, kappa * inv_kx_scale(ym, h, s0, s1)


def c2r_scale(ym: np.ndarray, h: int, w: int, s0: float | None = None, s1: float | None = None) -> np.ndarray:
    """|M| (|Re Y| + |Im Y|) of irfft2 on the kept modes (spectral_inverse; s0 / s1 default 1/HW, 2/HW): every twiddle
    has modulus 1, so sum_{kx,ky} c_ky (|Re Y| + |Im Y|), the same for every pixel: [B][O][H][W]."""
    c = _ky_factor(ym.shape[-1], 1.0 / (h * w) if s0 is None else s0, 2.0 / (h * w) if s1 is None else s1)
    tot = (_cabs(ym) * c).sum(axis=(-2, -1))
    return np.broadcast_to(tot[:, :, None, None], ym.shape[:2] + (h, w))


def block_out(ym, x, w0, bias, epi: str, kappa: float, pre_in=None, s0=None, s1=None):
    """Output stage of a Fourier block: lin = irfft2(pad(Y)) + W0 x (+ bias).  epi in gelu / save_pre (-> GELU(lin)),
    mul_dgelu (-> lin GELU'(pre_in)), plain (-> lin).  Returns (ref, bound, lin, lin_bound).
    lin: scale = c2r_scale + |W0| |x| + |b|.  GELU: 1.13 x the lin bound + the degree-8 fit's 2.7e-7 (+ the fp32
    rounding of the result, 2^-24 |ref|).  GELU'(pre_in) multiplies the lin bound by |GELU'(pre_in)| and adds
    |lin| DGELU_FIT."""
    h, w = x.shape[-2:]
    b = np.zeros(w0.shape[0]) if bias is None else bias
    lin = onp.spectral_inverse(ym, h, w, 12, 12, c0=s0, c1=s1) + onp.conv1x1(x, w0, b)
    scale = c2r_scale(ym, h, w, s0, s1) + onp.conv1x1(np.abs(x), np.abs(w0), np.abs(b))
    lin_bound = kappa * scale
    if epi in ("gelu", "save_pre"):
        ref = onp.gelu(lin)
        bound = SUP_DGELU * lin_bound + GELU_FIT[8] + 2.0 ** -24 * np.abs(ref)
    elif epi == "mul_dgelu":
        d = onp.dgelu(np.asarray(pre_in, np.float64))
        ref = lin * d
        bound = lin_bound * np.abs(d) + DGELU_FIT * np.abs(lin) + 2.0 ** -24 * np.abs(ref)
    else:
        ref, bound = lin, lin_bound
    return ref, bound, lin, lin_bound


def project(a, w1, b1, w2, b2, mask, kappa_fc1: float, gelu_degree: int):
    """preds = (fc2 . GELU . fc1)(a) * mask: (ref, bound).
    fc1: e1 = kappa_fc1 (|W1| |a| + |b1|) per hidden unit; GELU carries it as 1.13 e1.  fc2 adds these 128 independent
    rounding errors with the weights W2: LAMBDA sqrt(sum_j (W2_j 1.13 e1_j)^2), the Gaussian model of the module
    docstring (a linear sum |W2| e1 would be sqrt(128) looser and hide a defect in fc1).  The GELU fit's error is
    systematic, so it adds linearly: eps_fit sum_j |W2_j|; fc2's own rounding: kappa_fc2 (|W2| |GELU(z1)| + |b2|).
    Masked pixels must be exactly 0 (bound 0)."""
    w1m, w2m = w1.reshape(w1.shape[:2]), w2.reshape(w2.shape[:2])
    z1 = onp.conv1x1(a, w1m, b1)
    g = onp.gelu(z1)
    ref = onp.conv1x1(g, w2m, b2)
    e_g = SUP_DGELU * kappa_fc1 * onp.conv1x1(np.abs(a), np.abs(w1m), np.abs(b1))
    bound = LAMBDA * np.sqrt(np.einsum("cj,bjhw->bchw", w2m ** 2, e_g ** 2, optimize=True)) \
        + GELU_FIT[gelu_degree] * np.abs(w2m).sum(1)[None, :, None, None] \
        + KAPPA_FC2 * onp.conv1x1(np.abs(g), np.abs(w2m), np.abs(b2))
    m = mask[:, None] if mask.ndim == 3 else mask
    return ref * m, bound * m


def project_hidden(a, w1, b1, kappa_fc1: float):
    """GELU(z1), z1 = fc1(a), as the project backward recomputes it (degree-8 fit): (ref, bound), the bound carrying fc1's
    error through GELU (1.13 e_z1) plus the fit's 2.7e-7 and the fp32 rounding of the result.  The Q operand of the
    fc2.weight gradient."""
    w1m = w1.reshape(w1.shape[:2])
    g = onp.gelu(onp.conv1x1(a, w1m, b1))
    e_z1 = kappa_fc1 * onp.conv1x1(np.abs(a), np.abs(w1m), np.abs(b1))
    return g, SUP_DGELU * e_z1 + GELU_FIT[8] + 2.0 ** -24 * np.abs(g)


def project_bwd(a, dpreds, mask, pre, w1, b1, w2, kappa_fc1: float = KAPPA_FC1["grid"],
                kappa_da: float = KAPPA_DA["grid"], with_dz1: bool = False):
    """dpre = (W1^T ((W2^T (dpreds mask)) GELU'(z1))) GELU'(pre), the last block's adjoint through the projection:
    (ref, bound), the same rules on the adjoint: each product carries the bound of its factors (|x| e_y + |y| e_x), each
    contraction |W|^T (e) + kappa(n) |W|^T |.|, GELU' of a computed z1 moves by at most 0.8 e_z1 + its fit's error.
    kappa_fc1 / kappa_da are the kappas of the two contractions, z1 = W1 a + b1 and da = W1^T dz1 (KAPPA_FC1,
    KAPPA_DA: the grid kernel's FFMA chains by default, the tensor-core kernel's 3xTF32 / 2-pass GEMMs for 64 x 64).
    pre = None: no GELU'(pre) factor.  with_dz1: also (dz1_ref, dz1_bound), dz1 = (W2^T dpreds mask) GELU'(z1), the
    kernel's second output (the operand of the fc1 gradients)."""
    w1m, w2m = w1.reshape(w1.shape[:2]), w2.reshape(w2.shape[:2])
    m = mask[:, None] if mask.ndim == 3 else mask
    graw = dpreds * m
    z1 = onp.conv1x1(a, w1m, b1)
    e_z1 = kappa_fc1 * onp.conv1x1(np.abs(a), np.abs(w1m), np.abs(b1))
    d1 = onp.dgelu(z1)
    g2 = np.einsum("cj,bchw->bjhw", w2m, graw, optimize=True)
    s_g2 = np.einsum("cj,bchw->bjhw", np.abs(w2m), np.abs(graw), optimize=True)
    gz1 = g2 * d1
    e_gz1 = kappa(3) * s_g2 * np.abs(d1) + s_g2 * (SUP_D2GELU * e_z1 + DGELU_FIT)
    ga = np.einsum("ji,bjhw->bihw", w1m, gz1, optimize=True)
    e_ga = np.einsum("ji,bjhw->bihw", np.abs(w1m), e_gz1 + kappa_da * np.abs(gz1), optimize=True)
    if pre is None:
        ref, bound = ga, e_ga
    else:
        d = onp.dgelu(pre)
        ref = ga * d
        bound = e_ga * np.abs(d) + DGELU_FIT * np.abs(ga) + 2.0 ** -24 * np.abs(ref)
    return (ref, bound, gz1, e_gz1) if with_dz1 else (ref, bound)


# ------------------------------------------------------------------------------------------ backward reductions
# A weight gradient is a sum over samples and pixels, G[j][i] = sum_{b,pix} P[b][j][pix] Q[b][i][pix] (bias gradients:
# Q = 1), spread over CTAs, thread groups and a second reduce_partials launch.  Its rounding term is kappa(n) sum|P||Q|
# with n the LONGEST chain of additions any one term passes through, not the B H W term count: with the term count the
# bound is sqrt(#CTAs #groups) looser and a defect confined to one thread tile or one CTA's share stays under it.  Each
# chain below is read off the kernel's launch code, as a function of the batch (nb: the samples of one launch), the
# grid and, where the grid is capped by it, the SM count.  Where an operand carries its own bound (dz1, GELU(z1)), the
# propagation |Q|^T e_P + |P|^T e_Q is added (Outer).  The reductions' real errors cancel far more than sum|P||Q| allows
# for, so they use little of these bounds; a missing pixel group, sample or wrong column still exceeds them 80x to 1e5x
# in tests/test_backward_bounds_host.py.  Largest |err| / bound measured by tests/test_gpu_backward_bounds.py on an
# H100 80GB HBM3 (SXM, 700 W power limit), 22 configurations (64 x 64 both storage modes, B = 1 .. 256; 66 x 65,
# 25 x 127, 24 x 24 at B = 265):
#   fc2.weight 4.9e-4, fc2.bias 1.0e-3, fc1.bias 9.2e-4, fc1.weight 1.9e-3, w0.weight 3.6e-3, w0.bias 1.8e-3,
#   weights1 | weights2 0.14, fc0.weight 3.4e-3, fc0.bias 1.9e-3, d_inputs 0.13, d_case_params 2.1e-3;
#   the data path on the existing stage bounds: gm (fp32 DFT at (1/HW, 2/HW)) 0.070 (64 x 64), 0.21 (grids), ym (adjoint
#   mix, KAPPA_MIX) 0.12, z (inv_kx at (1, 1)) 0.060, dL/da0 (block_out PLAIN) 0.078.
def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def chain_reduce_partials(n_parts: int, n_launches: int = 1) -> int:
    """reduce_partials_kernel: thread (tx, ty) adds rows ty, ty + 32, .. (at most ceil(n / 32) into one of its four
    sums), the four sums pairwise (2), then the 32 row groups in order (31); a further batch chunk adds its sum to the
    gradient (+1 per launch after the first)."""
    return _cdiv(n_parts, 32) + 2 + 31 + (n_launches - 1)


def chain_chan_outer(nb: int, nj: int, n_launches: int = 1) -> int:
    """chan_outer_kernel<NJ, 32> (64 x 64) + reduce_partials: items = nb 4096 / PIX chunks on min(items, 296) CTAs; a
    thread adds PXG pixels of each of its ceil(items / grid) items in one FFMA chain, then the NG pixel groups' tiles are
    added in order.  NJ = 128 (fc1): NG = 2, PIX = 64, PXG = 32; NJ = 32 (w0): NG = 8, PIX = 128, PXG = 16."""
    ng, pix = 256 // nj, (64 if nj >= 128 else 128)
    items = nb * (4096 // pix)
    grid = min(items, 296)
    return _cdiv(items, grid) * (pix // ng) + (ng - 1) + chain_reduce_partials(grid, n_launches)


def chain_project_bwd_tc(nb: int, n_sm: int, n_launches: int = 1) -> int:
    """project_bwd_tc_kernel's fc2.weight / fc1.bias / fc2.bias partials + reduce_partials: 64 one-row tiles per sample
    on 2 min(ceil(32 nb), n_sm, 256) pipelines; per tile a sum over two rows (2, fc2.bias: in the thread's running sum),
    the halving transpose-reduction over 8 lanes (3), the four warps (3), then the pipeline's running total, one add per
    tile."""
    tiles = 64 * nb
    grid = min(_cdiv(tiles, 2), n_sm, 256)
    per_pipe = _cdiv(tiles, 2 * grid)
    return 2 * per_pipe + 8 + chain_reduce_partials(2 * grid, n_launches)


def chain_spectral_wgrad(b: int) -> int:
    """spectral_wgrad_kernel: warp w takes samples w, w + 4, .. (ceil(B / 4)); conj(x) g adds two FFMA chains of that
    length (2 ceil(B / 4) + 1), then the four warps (3)."""
    return 2 * _cdiv(b, 4) + 4


def chain_lift_bwd(b: int) -> int:
    """lift_bwd_kernel + lift_bwd_reduce (64 x 64): grid.y = min(B, 16) slices; a thread adds 16 terms per sample (four
    float4 groups, each a 4-FFMA chain) over ceil(B / grid.y) samples, the warp butterfly (5), the 8 warps (7), then the
    grid.y partial rows (grid.y).  The case-parameter columns (per-sample plane sums times params) are shorter."""
    gy = min(b, 16)
    return 16 * _cdiv(b, gy) + 12 + gy


# lift_bwd_data_kernel: d_inputs = 32 FFMA over the channels; d_case_params: a thread's 8-pixel sum (8), 32 FFMA over
# the channels, the warp butterfly (5) and 16 warps (15)
CHAIN_LIFT_DATA = {"d_inputs": 32, "d_case_params": 60}


def chain_grid_project_bwd(nb: int, hw: int, n_launches: int = 1) -> int:
    """grid_project_bwd_kernel + reduce_partials: nb ceil(hw / 32) 32-pixel tiles on min(tiles, 1024) CTAs, 32 FFMA per
    tile (fc2.bias: a 32-term sum per tile)"""
    tiles = nb * _cdiv(hw, 32)
    parts = min(tiles, 1024)
    return 32 * _cdiv(tiles, parts) + chain_reduce_partials(parts, n_launches)


def chain_grid_chan_outer(nb: int, hw: int, n_launches: int = 1) -> int:
    """grid_chan_outer_kernel + reduce_partials: 32-pixel tiles on min(tiles, 528) CTAs, 32 FFMA per tile"""
    tiles = nb * _cdiv(hw, 32)
    parts = min(tiles, 528)
    return 32 * _cdiv(tiles, parts) + chain_reduce_partials(parts, n_launches)


def chain_grid_lift_bwd(b: int, hw: int) -> int:
    """grid_lift_bwd_kernel + reduce_partials: min(B, 264) CTAs take ceil(B / parts) samples each; per sample a lane's
    ceil(hw / 32) FFMA, the warp butterfly (5) and one add into the CTA's running row"""
    parts = min(b, 264)
    return _cdiv(b, parts) * (_cdiv(hw, 32) + 6) + chain_reduce_partials(parts)


def chain_grid_lift_data(hw: int) -> dict:
    """grid_lift_bwd_kernel's data adjoint: d_inputs 32 FFMA; d_case_params a lane's ceil(hw / 32) pixels, the warp
    butterfly (5) and 32 FFMA over the channels"""
    return {"d_inputs": 32, "d_case_params": _cdiv(hw, 32) + 37}


class Outer:
    """G[j][i] = sum_{b,pix} P[b][j][pix] Q[b][i][pix] and the row sums r[j] = sum P[b][j][pix], accumulated over
    sample chunks (`add`), with their scales sum |P||Q| and sum |P| and the propagation of the operands' own bounds,
    |Q|^T e_P + |P|^T e_Q (row sums: sum e_P).  `weight(chain)` / `rowsum(chain)` give (ref, bound)."""

    def __init__(self):
        self.g = self.s = self.e = self.r = self.rs = self.re = 0.0

    def add(self, p, q, e_p=None, e_q=None):
        b, nj, ni = p.shape[0], p.shape[1], q.shape[1]
        p, q = p.reshape(b, nj, -1), q.reshape(b, ni, -1)
        ap, aq = np.abs(p), np.abs(q)
        self.g = self.g + np.einsum("bjn,bin->ji", p, q, optimize=True)
        self.s = self.s + np.einsum("bjn,bin->ji", ap, aq, optimize=True)
        self.r = self.r + p.sum(axis=(0, 2))
        self.rs = self.rs + ap.sum(axis=(0, 2))
        if e_p is not None:
            e_p = e_p.reshape(b, nj, -1)
            self.e = self.e + np.einsum("bjn,bin->ji", e_p, aq, optimize=True)
            self.re = self.re + e_p.sum(axis=(0, 2))
        if e_q is not None:
            self.e = self.e + np.einsum("bjn,bin->ji", ap, e_q.reshape(b, ni, -1), optimize=True)
        return self

    def weight(self, chain: int):
        return self.g, kappa(chain) * self.s + self.e

    def rowsum(self, chain: int):
        return self.r, kappa(chain) * self.rs + self.re


def spectral_wgrad(xm, gm, chain: int):
    """gW[i][o][kx][ky] = sum_b conj(X[b][i][kx][ky]) G[b][o][kx][ky]: (ref complex, bound for Re and Im), scale
    sum_b (|Re x| + |Im x|)(|Re g| + |Im g|)."""
    ref = np.einsum("bikl,bokl->iokl", np.conj(xm), gm, optimize=True)
    return ref, kappa(chain) * np.einsum("bikl,bokl->iokl", _cabs(xm), _cabs(gm), optimize=True)


def lift_data(da0, w_lift, chains: dict):
    """The lift's data adjoint from dL/da0 [B][32][H][W] and fc0.weight [32][5 + p] (columns u, v, mask, x, y, params):
    d_inputs = W[:, :2]^T da0 (scale |W|^T |da0|) and d_case_params[b][j] = sum_o W[o][5 + j] sum_pix da0[b][o] (scale
    sum_o |W| sum_pix |da0|): ((ref, bound), (ref, bound))."""
    w = w_lift.reshape(w_lift.shape[:2])
    wi, wp = w[:, :2], w[:, 5:]
    d_in = np.einsum("oc,bohw->bchw", wi, da0, optimize=True)
    s_in = np.einsum("oc,bohw->bchw", np.abs(wi), np.abs(da0), optimize=True)
    d_cp = np.einsum("oj,bo->bj", wp, da0.sum(axis=(2, 3)), optimize=True)
    s_cp = np.einsum("oj,bo->bj", np.abs(wp), np.abs(da0).sum(axis=(2, 3)), optimize=True)
    return (d_in, kappa(chains["d_inputs"]) * s_in), (d_cp, kappa(chains["d_case_params"]) * s_cp)


# ------------------------------------------------------------------------------------------ the checks
def bf16_interval(got: np.ndarray, ref: np.ndarray, bound: np.ndarray) -> np.ndarray:
    """Per element: the stored bf16 value `got` is the bf16 rounding of some value in [ref - bound, ref + bound].  The
    kernel rounds an fp32 value, and fp32-then-bf16 rounding (onp.bf16_round) is monotone, so this is exactly
    bf16(ref - bound) <= got <= bf16(ref + bound).  Returns the boolean mask of violations."""
    lo = onp.bf16_round(ref - bound)
    hi = onp.bf16_round(ref + bound)
    return ~((lo <= got) & (got <= hi))


def flip_share(got: np.ndarray, ref: np.ndarray) -> float:
    """share of bf16 stores that differ from the bf16 rounding of the float64 value"""
    return float((got != onp.bf16_round(ref)).mean())


PIXEL_AXES = ("sample", "channel", "h", "w")
MODE_AXES = ("kx", "ky", "sample", "channel")


def _groups(bad: np.ndarray, axes, tile) -> str:
    """How the failing elements group: per sample, per (sample, row) and per tile (`tile` = name -> function of the
    index arrays giving a tile id)."""
    idx = np.nonzero(bad)
    parts = []
    for name, fn in tile.items():
        keys = np.asarray(fn(*idx))
        ids, counts = np.unique(keys, return_counts=True, axis=0 if keys.ndim > 1 else None)
        top = np.argsort(-counts, kind="stable")[:6]
        parts.append(f"{len(counts)} {name}(s), most: " +
                     ", ".join(f"{tuple(int(v) for v in np.atleast_1d(ids[t]))}: {int(counts[t])}" for t in top))
    return "; ".join(parts)


def pixel_tiles(row_len: int = 64):
    """groupings of [B][C][H][W] failures: sample, (sample, row), (sample, 64-pixel tile of the flattened plane)"""
    return {"sample": lambda b, c, h, w: b,
            "(sample, row)": lambda b, c, h, w: np.stack([b, h], 1),
            "(sample, tile)": lambda b, c, h, w: np.stack([b, (h * row_len + w) // 64], 1)}


def mode_tiles():
    """groupings of [kx][ky][B][C] failures: mode, 128-sample tile, sample"""
    return {"mode (kx, ky)": lambda kx, ky, b, c: np.stack([kx, ky], 1),
            "128-sample tile": lambda kx, ky, b, c: b // 128,
            "sample": lambda kx, ky, b, c: b}


WEIGHT_AXES = ("row", "column")


def weight_tiles(thread_of):
    """groupings of [J][I] weight-gradient failures: (row, column) and the thread tile that owns the element
    (`thread_of(j, i)` -> thread id arrays, e.g. chan_outer's interleaved 8 x 4 tiles)"""
    return {"(row, column)": lambda j, i: np.stack([j, i], 1),
            "thread tile": lambda j, i: np.stack(thread_of(j, i), 1)}


def chan_outer_thread(nj: int, ni: int = 32):
    """chan_outer_kernel's thread (tj, ti) of G[j][i]: rows j = a NJ/8 + tj, columns i = c NI/4 + ti"""
    return lambda j, i: (j % (nj // 8), i % (ni // 4))


def grid_chan_outer_thread(nj: int, ni: int = 32):
    """grid_chan_outer_kernel's thread (tj, ti): a contiguous RJ x 4 block, RJ = NJ / 32"""
    return lambda j, i: (j // (nj // 32), i // 4)


def check(name: str, got, ref, bound, axes=PIXEL_AXES, tiles=None, bf16: bool = False) -> float:
    """Assert the per-element rule (bf16: the interval rule) and return max |got - ref| / bound (bf16: the share of
    stores that differ from the bf16 rounding of the float64 value, as rounding moves a store by up to half an ulp,
    which a ratio to the bound would not describe).  Complex arrays are
    checked on Re and Im with the same bound.  On failure the message names the worst element by `axes` and how the
    failing elements group (`tiles`)."""
    got = np.asarray(got)
    ref = np.asarray(ref)
    bound = np.broadcast_to(np.asarray(bound, np.float64), ref.shape)
    if np.iscomplexobj(ref):
        err = np.maximum(np.abs(got.real - ref.real), np.abs(got.imag - ref.imag))
    else:
        err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / bound)
    bad = bf16_interval(got, ref, bound) if bf16 else ~(err <= bound)
    worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    if bad.any():
        wb = np.unravel_index(int(np.argmax(np.where(bad, ratio, -1.0))), ratio.shape)
        where = ", ".join(f"{a}={int(i)}" for a, i in zip(axes, wb))
        msg = (f"{name}: {int(bad.sum())} of {bad.size} elements outside the bound; worst ({where}): got {got[wb]}, "
               f"ref {ref[wb]}, bound {float(bound[wb]):.3g}, |err|/bound {float(ratio[wb]):.3g}")
        if tiles:
            msg += "; " + _groups(bad, axes, tiles)
        raise AssertionError(msg)
    return flip_share(got, ref) if bf16 else float(ratio[worst])
