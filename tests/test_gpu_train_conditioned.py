"""The training pass stage by stage, each stage fed the GPU's own input to it (64x64: fno_forward_train +
fno_backward_inputs in both storage modes; other grids: fno_grid_forward_train + fno_grid_backward).

End-to-end gradient checks compare two forwards with different arithmetic, so in bf16 storage a few activations round to
different bf16 neighbours and the layers behind amplify those flips (DESIGN.md 5): such checks cannot be tighter than
~1e-2.  Conditioned on the saved tensors -- a_0..a_L (bf16 or fp32), pre_0..pre_{L-1} and the spectra xm[l] -- every
stage of the forward, and the whole backward, is a fixed computation with no rounding boundary in between: the backward
is a linear map of d(preds) evaluated in fp32.  So each is compared here with a float64 restatement fed the same saved
tensors (`oracle.fno_numpy.fno_vjp_saved` for the backward), at fp32-level bounds in BOTH storage modes.  The only
exception is a bf16 store, which must be the bf16 rounding of some value within the fp32 evaluation error of the float64
value (oracle.error_bounds.bf16_interval).

Every check is reported (`-s` prints the measured maxima) before it is asserted."""
import json

import numpy as np
import pytest
import torch
from scipy.special import erf

from cfdbench_b200 import synth
from oracle import error_bounds as eb
from oracle import fno_numpy as onp

from test_gpu_fused import assert_within_flip_ambiguity

pytestmark = pytest.mark.gpu

CHUNK_EDGES = (0, 31, 32, 63, 64)   # first / last samples of the project backward's 32-sample chunks
BARS = {"a0": 2e-6, "xm": 2e-6, "pre": 3e-6, "act": 1e-6, "preds": 3e-6}   # forward stages, per-sample max rel L2


def backward_bar(depth: int, what: str) -> float:
    """Relative L2 bar of the backward against fno_vjp_saved.  Each Fourier block's adjoint runs the arithmetic of a
    forward block (DFT, mode mix, inverse DFT, 1x1 conv on 3xTF32 tensor cores), whose error given its input is
    5e-7 .. 1e-6 (the pre[l] checks), and these errors add up along the chain: the measured maxima of the parameter
    gradients and d_inputs on the H100 are 2.1e-6 at depth 1, 6.3e-6 at depth 4 and 1.2e-5 at depth 8, about 1.4e-6
    per block.  The bar is 2.5e-6 per block plus the projection and the lift.  d_case_params is a per-sample sum of
    dL/da0 over all pixels, which cancels: its relative error is that of dL/da0 times the cancellation ratio (measured
    up to 1.3e-5 at depth 4 over 256 samples, 1.7e-5 at depth 8), so its bar is twice as wide."""
    return (2.0 if what == "d_case_params" else 1.0) * 2.5e-6 * (depth + 1)

# grid, storage, depth, p, B -- each row for a reason:
CONFIGS = [
    # one sample: chan_outer below its 296-CTA cap, lift_bwd grid.y = 1, 3 of 4 spectral_wgrad warps idle
    pytest.param("cavity", "float32", 4, 5, 1, id="cavity-fp32-L4-p5-B1"),
    pytest.param("cavity", "bfloat16", 4, 5, 1, id="cavity-bf16-L4-p5-B1"),
    # project-backward chunks 32 + 1, masked pixels
    pytest.param("cylinder", "float32", 4, 8, 33, id="cylinder-fp32-L4-p8-B33"),
    pytest.param("cylinder", "bfloat16", 4, 8, 33, id="cylinder-bf16-L4-p8-B33"),
    # a single block: the PLAIN epilogue right after the project backward, no case parameters
    pytest.param("cavity", "float32", 1, 0, 3, id="cavity-fp32-L1-p0-B3"),
    # FNO_MAX_LAYERS, kMaxCaseParams, ragged chunk tail
    pytest.param("cavity", "float32", 8, 16, 70, id="cavity-fp32-L8-p16-B70"),
    pytest.param("cavity", "bfloat16", 8, 16, 70, id="cavity-bf16-L8-p16-B70"),
    # the training batch bench.py times
    pytest.param("cavity", "bfloat16", 4, 5, 256, id="cavity-bf16-L4-p5-B256"),
    # grid path: grid_chan_outer, grid_lift_bwd
    pytest.param("tube", "float32", 4, 5, 33, id="tube66x65-fp32-L4-p5-B33"),
    # the grid range's ends, p = 16 on the grid lift backward
    pytest.param((128, 128), "float32", 2, 16, 3, id="grid128x128-fp32-L2-p16-B3"),
    pytest.param((24, 24), "float32", 1, 5, 70, id="grid24x24-fp32-L1-p5-B70"),
]


def _model(sd, p, depth, act):
    from cfdbench_b200 import Fno2d, loss_name_to_fn
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=depth, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m


def _batch(seed, b, where, p):
    """inputs / case_params / mask for `where` = a synth problem or an (H, W) grid (ones with wall rows / inlet column
    zeroed), with p case parameters."""
    rng = np.random.default_rng(seed)
    if isinstance(where, str):
        bt = synth.make_batch(seed, b, where, with_label=False)
    else:
        gh, gw = where
        mask = np.ones((b, 1, gh, gw), np.float32)
        mask[:, :, 0, :] = mask[:, :, gh - 1, :] = mask[:, :, :, 0] = 0.0
        bt = dict(inputs=np.clip(rng.standard_normal((b, 2, gh, gw)), -3, 3).astype(np.float32), mask=mask)
    if "case_params" not in bt or bt["case_params"].shape[1] != p:
        bt["case_params"] = rng.standard_normal((b, p)).astype(np.float32)
    return bt


def _upstream(seed, shape):
    """Random d(preds) with per-sample scales spread over 1.5 decades; the project-backward chunk edges and the last
    sample carry the largest weights, so that a lost or duplicated edge sample shows in the parameter gradients."""
    rng = np.random.default_rng(seed)
    b = shape[0]
    scale = 10.0 ** rng.uniform(-1.5, 0.0, b)
    scale[[i for i in CHUNK_EDGES + (b - 1,) if i < b]] = 3.0
    return (rng.standard_normal(shape) * scale[:, None, None, None]).astype(np.float32)


def _f64(t):
    t = t.detach().cpu()
    if t.is_complex():
        return t.to(torch.complex128).numpy()
    return t.double().numpy()


def _max_rel(got, ref):
    """max over samples (axis 0) of the relative L2 error."""
    b = ref.shape[0]
    d = np.linalg.norm((got - ref).reshape(b, -1), axis=1)
    return float(np.max(d / np.linalg.norm(ref.reshape(b, -1), axis=1)))


def _rel(got, ref):
    return float(np.linalg.norm(got - ref) / np.linalg.norm(ref))


def _gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def _bf16_key(x):
    """Integer order of bf16 values: adjacent bf16 numbers differ by 1 (+0 and -0 both map to 0)."""
    u = (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) >> np.uint32(16)).astype(np.int64)
    return np.where(u & 0x8000, -(u & 0x7FFF), u)


def _bf16_store_errors(got, ref64, bound):
    """A bf16 store against the float64 value: (largest distance in bf16 ulps from the float64 value rounded to bf16,
    share of elements that differ from it, number of elements that are not the bf16 rounding of any value within `bound`
    of the float64 value, where `bound` bounds the fp32 evaluation error of the stored value).  `got` holds the stored
    bf16 values (exact in float64)."""
    steps = np.abs(_bf16_key(got) - _bf16_key(onp.bf16_round(ref64)))
    return int(steps.max()), float((steps != 0).mean()), int(eb.bf16_interval(got, ref64, bound).sum())


def _project(sd, a, mask, chunk=32):
    out = np.empty((a.shape[0], 2) + a.shape[2:])
    for b0 in range(0, a.shape[0], chunk):
        z1 = onp.conv1x1(a[b0:b0 + chunk], sd["fc1.weight"], sd["fc1.bias"])
        out[b0:b0 + chunk] = onp.conv1x1(_gelu(z1), sd["fc2.weight"], sd["fc2.bias"])
    return out * mask


def _run_native(m, bt, gpreds):
    """forward_train + backward through the module's own native calls: (preds, saved tensors, gradients in parameter
    order, d_inputs, d_case_params), all still on the GPU."""
    x, cp, mask4 = m._prep_inputs(*(torch.from_numpy(bt[k]).cuda() for k in ("inputs", "case_params", "mask")))
    preds, saved = m._native_forward_train(x, mask4, cp)
    d_in, d_cp = torch.empty_like(x), torch.empty_like(cp)
    grads = m._native_backward(x, mask4, cp, torch.from_numpy(gpreds).cuda(), saved, True, d_in, d_cp)
    torch.cuda.synchronize()
    return preds, saved, grads, d_in, d_cp


def _report(what, errs):
    print(f"\n[{what}] " + json.dumps({k: (float(f"{v:.3g}") if isinstance(v, float) else v) for k, v in errs.items()}))


@pytest.mark.parametrize("where,act,depth,p,b", CONFIGS)
def test_training_pass_stages_against_float64_conditioned_on_saved_tensors(where, act, depth, p, b, request):
    seed = 1000 * depth + 10 * p + b
    sd = synth.make_state_dict(seed, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(seed + 1, b, where, p)
    gh, gw = bt["inputs"].shape[-2:]
    gpreds = _upstream(seed + 2, (b, 2, gh, gw))
    m = _model(sd, p, depth, act)
    preds, (_, acts_g, pres_g, xms_g), grads_g, d_in_g, d_cp_g = _run_native(m, bt, gpreds)
    bf = act == "bfloat16"
    assert acts_g[0].dtype == (torch.bfloat16 if bf else torch.float32)
    mask = bt["mask"].astype(np.float64)
    acts = [_f64(a) for a in acts_g]
    pres = [_f64(t) for t in pres_g]
    errs, fails = {}, []

    def check(name, value, bar):
        errs[name] = value
        if not value <= bar:
            fails.append((name, value, bar))

    def check_store(name, got, ref64, eval_err):
        if bf:
            ulps, share, outside = _bf16_store_errors(got, ref64, eval_err)
            errs[name + ".ulps"], errs[name + ".flip_share"], errs[name + ".outside"] = ulps, share, outside
            if outside:
                fails.append((name, ulps, share, outside))
        else:
            check(name, _max_rel(got, ref64), BARS["a0" if name == "a0" else "act"])

    # ---- forward stages
    feats = onp.lift_features(bt["inputs"], bt["case_params"], mask)
    lift = onp.conv1x1(feats, sd["fc0.weight"], sd["fc0.bias"])
    # a0 is a (5 + p)-term fp32 dot product: where its terms cancel, the fp32 evaluation error (<= (5 + p + 1) 2^-24 the
    # sum of the terms' magnitudes) is many ulps of the small result, so a0's bf16 store gets that allowance
    eval_err = (6 + p) * 2.0 ** -24 * onp.conv1x1(np.abs(feats), np.abs(sd["fc0.weight"]), np.abs(sd["fc0.bias"]))
    check_store("a0", acts[0], lift, eval_err)
    for l in range(depth):
        xm = onp.spectral_modes(acts[l], 12, 12)                               # [B][32][24][12]
        xm_g = _f64(xms_g[l]).reshape(24, 12, b, 32).transpose(2, 3, 0, 1)   # mode-major [288][B][32] -> the same
        check(f"xm[{l}]", _max_rel(xm_g, xm), BARS["xm"])
        wt = onp.stack_weights(sd[f"blocks.{l}.conv0.weights1"], sd[f"blocks.{l}.conv0.weights2"])
        pre = onp.spectral_inverse(np.einsum("bikl,iokl->bokl", xm, wt, optimize=True), gh, gw, 12, 12) \
            + onp.conv1x1(acts[l], sd[f"blocks.{l}.w0.weight"], sd[f"blocks.{l}.w0.bias"])
        check(f"pre[{l}]", _max_rel(pres[l], pre), BARS["pre"])
        # the GELU of the saved fp32 pre-activation: the degree-8 fit's error and the fp32 rounding of its result
        ref_act = _gelu(pres[l])
        check_store(f"act[{l + 1}]", acts[l + 1], ref_act, eb.GELU_FIT[8] + 2.0 ** -24 * np.abs(ref_act))
    preds_np = _f64(preds)
    preds_ref = _project(sd, acts[depth], mask)
    if bf:
        # project_tc_kernel<bf16> evaluates its GELUs with the degree-5 fit (fno_common.cuh: within 6.4e-7 abs of the
        # float64 GELU), which fc2 sums over 128 hidden units: an absolute error per output channel, which is most of
        # the relative error where the predictions are small (measured 5.7e-5 relative at |preds| ~ 6e-3, 0.14 of this
        # bound; the fp32 kernel on the same activations: 7e-7)
        gelu_err = 6.4e-7 * np.abs(sd["fc2.weight"].reshape(2, -1)).sum(1)[None, :, None, None]
        ratio = np.abs(preds_np - preds_ref) / (gelu_err + BARS["preds"] * np.abs(preds_ref))
        check("preds.bound_ratio", float(ratio[np.broadcast_to(mask, ratio.shape) > 0].max()), 1.0)
    else:
        check("preds", _max_rel(preds_np, preds_ref), BARS["preds"])
    check("preds.masked_max_abs", float(np.abs(preds_np * (1.0 - mask)).max()), 0.0)

    # ---- backward against the float64 adjoint through the same saved tensors
    ref, d_in_ref, d_cp_ref = onp.fno_vjp_saved(sd, bt["inputs"], bt["case_params"], mask, gpreds, acts, pres)
    del acts, pres
    names = [k for k, _ in m.named_parameters()]
    assert set(names) == set(ref)
    grad_errs = {k: _rel(_f64(g), ref[k]) for k, g in zip(names, grads_g)}
    worst = max(grad_errs, key=grad_errs.get)
    bar = backward_bar(depth, "grad")
    check("grad.max", grad_errs[worst], bar)
    errs["grad.worst"] = worst
    for k, e in grad_errs.items():
        if not e <= bar:
            fails.append((k, e, bar))
    check("d_inputs", _max_rel(_f64(d_in_g), d_in_ref), backward_bar(depth, "d_inputs"))
    if p > 0:
        d_cp, bar = _f64(d_cp_g), backward_bar(depth, "d_case_params")
        check("d_case_params", _max_rel(d_cp, d_cp_ref), bar)
        check("d_case_params.column_max", _max_rel(d_cp.T, d_cp_ref.T), bar)   # every column, p = 16 too
    _report(request.node.callspec.id, errs)
    assert not fails, fails


@pytest.mark.parametrize("act", ["float32", "bfloat16"])
def test_gradients_are_additive_over_batch_splits(act):
    """The parameter gradients of 70 samples equal the sum of those of samples [0:33] and [33:70] (the project backward's
    chunks are 32 + 32 + 6 vs 32 + 1 and 32 + 5): a lost or double-counted sample would show at the 1e-2 level."""
    p, depth, b = 5, 4, 70
    sd = synth.make_state_dict(7, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(8, b, "cavity", p)
    gpreds = _upstream(9, (b, 2, 64, 64))
    m = _model(sd, p, depth, act)
    whole = _run_native(m, bt, gpreds)
    parts = [_run_native(m, {k: v[sl] for k, v in bt.items()}, gpreds[sl]) for sl in (slice(0, 33), slice(33, 70))]
    errs = {}
    for i, (k, _) in enumerate(m.named_parameters()):
        total = _f64(parts[0][2][i]) + _f64(parts[1][2][i])
        errs[k] = _rel(_f64(whole[2][i]), total)
    # per-sample quantities do not depend on the batch the sample travels in
    d_in = torch.cat([parts[0][3], parts[1][3]])
    d_cp = torch.cat([parts[0][4], parts[1][4]])
    errs["d_inputs"] = _max_rel(_f64(whole[3]), _f64(d_in))
    errs["d_case_params"] = _max_rel(_f64(whole[4]), _f64(d_cp))
    _report(f"additivity-{act}", {"max": max(errs.values()), "worst": max(errs, key=errs.get)})
    for k, e in errs.items():
        assert e <= 1e-6, (k, e)


def test_autograd_path_equals_the_direct_native_calls():
    """`(m(...)["preds"] * gpreds).sum().backward()` -- the path users run -- gives the gradients of the direct
    _native_forward_train / _native_backward calls the tests above check, bit for bit."""
    p, depth, b = 8, 4, 33
    sd = synth.make_state_dict(11, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(12, b, "cylinder", p)
    gpreds = _upstream(13, (b, 2, 64, 64))
    m = _model(sd, p, depth, "bfloat16")
    _, _, grads, d_in, d_cp = _run_native(m, bt, gpreds)
    x = torch.from_numpy(bt["inputs"]).cuda().requires_grad_(True)
    cp = torch.from_numpy(bt["case_params"]).cuda().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    (m(inputs=x, case_params=cp, mask=torch.from_numpy(bt["mask"]).cuda())["preds"]
     * torch.from_numpy(gpreds).cuda()).sum().backward()
    for (k, prm), g in zip(m.named_parameters(), grads):
        assert torch.equal(prm.grad, g), k
    assert torch.equal(x.grad, d_in) and torch.equal(cp.grad, d_cp)


# ------------------------------------------------------------------------------ inference at depths other than 4
@pytest.mark.parametrize("depth", [1, 8])
def test_inference_at_depth_1_and_8_fp32(depth):
    """generate and the graph-replayed generate_many at p = 16 against the float64 oracle, per sample."""
    p, b = 16, 3
    sd = synth.make_state_dict(20 + depth, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(30 + depth, b, "cylinder", p)
    m = _model(sd, p, depth, "float32")
    assert m.graph_rollout
    x, cp, mk = (torch.from_numpy(bt[k]).cuda() for k in ("inputs", "case_params", "mask"))
    with torch.no_grad():
        y = m.generate(x, cp, mk)
    seq = m.generate_many(x, cp, mk, 2)
    assert torch.equal(seq[0], y)
    e1 = _max_rel(_f64(y), onp.fno_forward(sd, bt["inputs"], bt["case_params"], bt["mask"])["preds"])
    e2 = _max_rel(_f64(seq[1]), onp.fno_forward(sd, y.cpu().numpy(), bt["case_params"], bt["mask"])["preds"])
    _report(f"inference-fp32-L{depth}", {"step1": e1, "step2": e2})
    assert e1 <= 1e-5 and e2 <= 1e-5, (e1, e2)


@pytest.mark.parametrize("depth", [1, 8])
def test_inference_at_depth_1_and_8_bf16(depth):
    """bf16 storage, p = 16: the fused path against the two bf16-boundary oracles, and against the unfused path."""
    p, b = 16, 3
    sd = synth.make_state_dict(40 + depth, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(50 + depth, b, "cylinder", p)
    m = _model(sd, p, depth, "bfloat16")
    assert m.fused_block and m.graph_rollout
    x, cp, mk = (torch.from_numpy(bt[k]).cuda() for k in ("inputs", "case_params", "mask"))
    with torch.no_grad():
        y = m.generate(x, cp, mk)
    seq = m.generate_many(x, cp, mk, 2)
    assert torch.equal(seq[0], y)
    got = y.cpu().numpy()
    floor, e_t, e_n = assert_within_flip_ambiguity(got, sd, bt, f"depth {depth}")
    step2 = dict(inputs=got, case_params=bt["case_params"], mask=bt["mask"])   # teacher-forced from the GPU's step 1
    floor2, e_t2, e_n2 = assert_within_flip_ambiguity(seq[1].cpu().numpy(), sd, step2, f"depth {depth}, step 2")
    m2 = _model(sd, p, depth, "bfloat16")
    m2.fused_block = False
    with torch.no_grad():
        unfused = m2.generate(x, cp, mk).cpu().numpy()
    e_u = onp.rel_l2(got.astype(np.float64), unfused.astype(np.float64))
    _report(f"inference-bf16-L{depth}", {"floor": floor, "vs_torch16": e_t, "vs_numpy16": e_n, "step2_floor": floor2,
                                         "step2_vs_torch16": e_t2, "step2_vs_numpy16": e_n2, "fused_vs_unfused": e_u})
    assert e_u < 2.0 * floor + 2e-5, (e_u, floor)
