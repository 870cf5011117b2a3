"""Every backward kernel checked ELEMENT BY ELEMENT against float64 fed the GPU's own input to its stage, with the
bounds of oracle/error_bounds.py, at the batches where each kernel's schedule changes (from the device's SM count).

One forward_train and one backward (fno_backward_inputs / fno_grid_backward, d_inputs and d_case_params requested) run
on scratch this test owns, built as Fno2d._native_backward builds it.  The drivers ping-pong the two d buffers, so after
the call, with cur = L mod 2: d[1 - cur] holds dpre_0 (for L = 1: the project backward's output for all samples), dz1
the last 32-sample chunk's dz1, gm the DFT of dpre_0 at (1/HW, 2/HW) (mode-major [288][B][32]), the workspace's ym and
z the adjoint mix of gm and its inverse kx at (1, 1), and d[cur] dL/da0.  Checked here:
  * the project backward: dpre_{L-1} (L = 1), the last chunk's dz1, and fc2.weight, fc1.bias, fc2.bias, fc1.weight from
    the saved a_L and dpreds, accumulated over all chunks;
  * layer 0's data path: gm, ym, z and dL/da0 (block_out PLAIN with W0 untransposed);
  * layer 0's w0.weight / w0.bias and weights1 / weights2 (spectral_wgrad + unpack);
  * fc0.weight / fc0.bias, d_inputs and d_case_params from dL/da0.
Layers >= 1 run the same kernels on other pointers; test_gpu_train_conditioned covers them.  The float64 references
are formed per 32-sample chunk.  `-s` prints each stage's max |err| / bound."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from oracle import error_bounds as eb
from oracle import fno_numpy as onp

from test_gpu_train_conditioned import _batch, _model, _upstream

pytestmark = pytest.mark.gpu

CHUNK = 32


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _batch_for(case):
    """64 x 64 batches where a backward kernel's schedule changes"""
    return {"one": 1,                                  # every reduction below its cap, 3 of 4 spectral_wgrad warps idle
            "prefetch": 2 * _n_sm() // 64 + 1,         # project_bwd's tiles exceed two per CTA; chan_outer(fc1) > 296
            "co_wrap": 296 // 32 + 1,                  # chan_outer(w0)'s 296 CTAs wrap
            "sw_wrap": 12 + 1,                         # spectral_wgrad's 12-deep queue wraps
            "lb_wrap": 16 + 1,                         # lift_bwd's 16 slices take a second sample
            "chunks": CHUNK + 1}[case]                 # project chunks 32 + 1: the fc1 / fc2 gradients accumulate


# storage, case / batch, depth, p
CONFIGS = [pytest.param(act, case, 1, p, id=f"{act}-{case}-p{p}")
           for act in ("float32", "bfloat16")
           for case, p in (("one", 5), ("prefetch", 5), ("co_wrap", 0), ("sw_wrap", 5), ("lb_wrap", 8), ("chunks", 5))]
CONFIGS += [pytest.param(act, 70, 4, 16, id=f"{act}-B70-L4-p16") for act in ("float32", "bfloat16")]   # ragged chunks
CONFIGS += [pytest.param("bfloat16", 256, 1, 5, id="bfloat16-B256"),                       # the training batch
            pytest.param("float32", 256, 1, 5, id="float32-B256")]

GRID_CONFIGS = [
    pytest.param((66, 65), 1, 1, 5, id="66x65-B1"),
    pytest.param((66, 65), 4, 1, 5, id="66x65-B4"),     # grid_chan_outer passes its 528 parts
    pytest.param((66, 65), 8, 1, 0, id="66x65-B8-p0"),  # grid_project_bwd passes its 1024 parts
    pytest.param((66, 65), 33, 2, 8, id="66x65-B33-L2"),
    pytest.param((25, 127), 3, 1, 16, id="25x127-B3"),  # odd H W
    pytest.param((24, 24), 265, 1, 5, id="24x24-B265"),  # grid_lift_bwd passes its 264 parts
]


def _h(t):
    t = t.detach().cpu()
    if t.dtype == torch.bfloat16:
        t = t.float()
    return t.to(torch.complex128).numpy() if t.is_complex() else t.double().numpy()


def _run(m, bt, gpreds):
    """forward_train + one backward into scratch owned here; returns every buffer the checks read, on the host"""
    from cfdbench_b200.fno2d import _ptr
    x, cp, mask4 = m._prep_inputs(*(torch.from_numpy(bt[k]).cuda() for k in ("inputs", "case_params", "mask")))
    b = x.shape[0]
    _, saved = m._native_forward_train(x, mask4, cp)
    pk = m._pack(need_bwd=True)
    route = m._route(*x.shape[-2:])
    ws, wbufs = m._workspace(b, route)
    _, views, g = m._grad_buffers()
    sc, sbufs = m._bwd_scratch(b, route)
    d_in = torch.empty_like(x)
    d_cp = torch.empty_like(cp) if m.n_case_params else None
    dp = torch.from_numpy(gpreds).cuda()
    route.call("backward", C.byref(m._coords(pk, route.gh, route.gw)[0]), C.byref(pk["struct_bwd"]), x.data_ptr(),
               mask4.data_ptr(), cp.data_ptr(), dp.data_ptr(), C.byref(saved[0]), C.byref(g), C.byref(sc), C.byref(ws),
               d_in.data_ptr(), _ptr(d_cp), b, m._stream())
    torch.cuda.synchronize()
    _, acts, pres, xms = saved
    L = m.num_layers
    cur = L % 2
    gh, gw = route.gh, route.gw
    z = _h(wbufs["z"]).reshape(b, gh, 12, 2, 32)
    out = dict(a0=_h(acts[0]), aL=_h(acts[L]), pre=_h(pres[L - 1]), xm0=_h(xms[0]),
               dpre0=_h(sbufs[f"d{1 - cur}"]), da0=_h(sbufs[f"d{cur}"]), dz1=_h(sbufs["dz1"]), gm=_h(sbufs["gm"]),
               ym=_h(wbufs["ym"]), z=(z[:, :, :, 0] + 1j * z[:, :, :, 1]).transpose(0, 3, 1, 2),
               grads={k: _h(v) for k, v in views.items()}, d_in=_h(d_in), d_cp=None if d_cp is None else _h(d_cp))
    return out


def _modes(a, b):
    """mode-major [288][B][32] -> [B][32][24][12]"""
    return a.reshape(24, 12, b, 32).transpose(2, 3, 0, 1)


def _check_all(where, act, b, depth, p, name):
    t0 = time.time()
    seed = 7000 + 100 * depth + 10 * p + b
    sd = synth.make_state_dict(seed, n_params=p, depth=depth, spectral_gain=50.0)
    bt = _batch(seed + 1, b, where, p)
    gh, gw = bt["inputs"].shape[-2:]
    hw = gh * gw
    grid = (gh, gw) != (64, 64)
    gpreds = _upstream(seed + 2, (b, 2, gh, gw))
    m = _model(sd, p, depth, act)
    g = _run(m, bt, gpreds)
    mask = bt["mask"].reshape(b, gh, gw).astype(np.float64)
    storage = "grid" if grid else ("f32" if act == "float32" else "bf16")
    k_fc1, k_da = eb.KAPPA_FC1[storage], eb.KAPPA_DA["grid" if grid else "tc"]
    ptiles = eb.pixel_tiles(gw)
    r = {}
    n_chunks = -(-b // CHUNK)

    # ---- project backward, per 32-sample chunk: dpre (L = 1), the last chunk's dz1, the fc1 / fc2 reductions
    w1, b1, w2 = sd["fc1.weight"], sd["fc1.bias"], sd["fc2.weight"]
    fc1w, fc2w = eb.Outer(), eb.Outer()
    for b0 in range(0, b, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        nb = min(CHUNK, b - b0)
        a = g["aL"][sl]
        ref, bound, dz1, e_dz1 = eb.project_bwd(a, gpreds[sl].astype(np.float64), mask[sl],
                                                g["pre"][sl], w1, b1, w2, k_fc1, k_da,
                                                with_dz1=True)
        if depth == 1:
            r["dpre"] = max(r.get("dpre", 0.0), eb.check(f"{name} dpre[{b0}:]", g["dpre0"][sl], ref, bound,
                                                          tiles=ptiles))
        if b0 + nb == b:
            r["dz1"] = eb.check(f"{name} dz1 (last chunk)", g["dz1"][:nb], dz1, e_dz1, tiles=ptiles)
        graw = gpreds[sl].astype(np.float64) * mask[sl][:, None]
        hid, e_hid = eb.project_hidden(a, w1, b1, k_fc1)
        fc2w.add(graw, hid, e_q=e_hid)
        fc1w.add(dz1, a, e_p=e_dz1)
        del ref, bound, dz1, e_dz1, hid, e_hid
    gr = g["grads"]
    if grid:
        ch_pb = eb.chain_grid_project_bwd(min(b, CHUNK), hw, n_chunks)
        ch_fc1 = eb.chain_grid_chan_outer(min(b, CHUNK), hw, n_chunks)
        th_fc1 = eb.grid_chan_outer_thread(128)
    else:
        ch_pb = eb.chain_project_bwd_tc(min(b, CHUNK), _n_sm(), n_chunks)
        ch_fc1 = eb.chain_chan_outer(min(b, CHUNK), 128, n_chunks)
        th_fc1 = eb.chan_outer_thread(128)
    ref, bound = fc2w.weight(ch_pb)
    r["fc2.weight"] = eb.check(f"{name} fc2.weight", gr["fc2.weight"].reshape(2, 128), ref, bound, axes=eb.WEIGHT_AXES,
                               tiles={"(row, column)": lambda j, i: np.stack([j, i], 1)})
    ref, bound = fc2w.rowsum(ch_pb)
    r["fc2.bias"] = eb.check(f"{name} fc2.bias", gr["fc2.bias"], ref, bound, axes=("column",))
    ref, bound = fc1w.rowsum(ch_pb)
    r["fc1.bias"] = eb.check(f"{name} fc1.bias", gr["fc1.bias"], ref, bound, axes=("column",))
    ref, bound = fc1w.weight(ch_fc1)
    r["fc1.weight"] = eb.check(f"{name} fc1.weight", gr["fc1.weight"].reshape(128, 32), ref, bound,
                               axes=eb.WEIGHT_AXES, tiles=eb.weight_tiles(th_fc1))
    del fc1w, fc2w

    # ---- layer 0's data path, each stage fed the GPU's own input
    dpre0 = g["dpre0"]
    inv = 1.0 / hw
    kdft = eb.kappa_dft_f32(gh, gw)
    mt = eb.mode_tiles()
    gm = _modes(g["gm"], b)
    gm_ref = np.empty_like(gm)
    for b0 in range(0, b, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        ref, bound = eb.dft(dpre0[sl], kdft, s0=inv, s1=2 * inv)
        gm_ref[sl] = ref
        r["gm"] = max(r.get("gm", 0.0), eb.check(f"{name} gm", g["gm"].reshape(24, 12, b, 32)[:, :, sl],
                                                  ref.transpose(2, 3, 0, 1), bound.transpose(2, 3, 0, 1),
                                                  axes=eb.MODE_AXES, tiles=mt))
    wt = onp.stack_weights(sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"])
    ref, bound = eb.mode_mix(gm, np.conj(wt).transpose(1, 0, 2, 3))
    r["ym"] = eb.check(f"{name} ym (adjoint mix)", g["ym"].reshape(24, 12, b, 32), ref.transpose(2, 3, 0, 1),
                       bound.transpose(2, 3, 0, 1), axes=eb.MODE_AXES, tiles=mt)
    ym = _modes(g["ym"], b)
    ref, bound = eb.inv_kx(ym, gh, 1.0, 1.0)
    r["z"] = eb.check(f"{name} z (inv_kx at (1, 1))", g["z"], ref, bound, axes=("sample", "channel", "h", "ky"),
                      tiles=eb.pixel_tiles(12))
    w0 = sd["blocks.0.w0.weight"].reshape(32, 32)
    k_bo = eb.KAPPA_GRID_BLOCK_OUT if grid else eb.KAPPA_BLOCK_TC
    for b0 in range(0, b, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        ref, bound, _, _ = eb.block_out(ym[sl], dpre0[sl], np.ascontiguousarray(w0.T), None, "plain", k_bo, s0=1.0,
                                        s1=1.0)
        r["da0"] = max(r.get("da0", 0.0), eb.check(f"{name} da0[{b0}:]", g["da0"][sl], ref, bound, tiles=ptiles))

    # ---- layer 0's weight gradients
    w0g = eb.Outer()
    for b0 in range(0, b, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        w0g.add(dpre0[sl], g["a0"][sl])
    if grid:
        ch_w0, th_w0 = eb.chain_grid_chan_outer(b, hw), eb.grid_chan_outer_thread(32)
    else:
        ch_w0, th_w0 = eb.chain_chan_outer(b, 32), eb.chan_outer_thread(32)
    ref, bound = w0g.weight(ch_w0)
    r["w0.weight"] = eb.check(f"{name} w0.weight", gr["blocks.0.w0.weight"].reshape(32, 32), ref, bound,
                              axes=eb.WEIGHT_AXES, tiles=eb.weight_tiles(th_w0))
    ref, bound = w0g.rowsum(ch_w0)
    r["w0.bias"] = eb.check(f"{name} w0.bias", gr["blocks.0.w0.bias"], ref, bound, axes=("column",))
    xm0 = _modes(g["xm0"], b)
    ref, bound = eb.spectral_wgrad(xm0, gm, eb.chain_spectral_wgrad(b))
    sw = np.concatenate([gr["blocks.0.conv0.weights1"], gr["blocks.0.conv0.weights2"]], axis=2)
    r["weights1|2"] = eb.check(f"{name} weights1 | weights2", sw, ref, bound, axes=("in", "out", "kx", "ky"),
                               tiles={"mode (kx, ky)": lambda i, o, kx, ky: np.stack([kx, ky], 1)})

    # ---- the lift's gradients from dL/da0
    da0 = g["da0"]
    lift = eb.Outer()
    for b0 in range(0, b, CHUNK):
        sl = slice(b0, b0 + CHUNK)
        lift.add(da0[sl], onp.lift_features(bt["inputs"][sl], bt["case_params"][sl], mask[sl]))
    ch_lb = eb.chain_grid_lift_bwd(b, hw) if grid else eb.chain_lift_bwd(b)
    ref, bound = lift.weight(ch_lb)
    r["fc0.weight"] = eb.check(f"{name} fc0.weight", gr["fc0.weight"].reshape(32, 5 + p), ref, bound,
                               axes=eb.WEIGHT_AXES, tiles={"column": lambda j, i: i})
    ref, bound = lift.rowsum(ch_lb)
    r["fc0.bias"] = eb.check(f"{name} fc0.bias", gr["fc0.bias"], ref, bound, axes=("column",))
    chains = eb.chain_grid_lift_data(hw) if grid else eb.CHAIN_LIFT_DATA
    (di, di_b), (dc, dc_b) = eb.lift_data(da0, sd["fc0.weight"], chains)
    r["d_inputs"] = eb.check(f"{name} d_inputs", g["d_in"], di, di_b, tiles=ptiles)
    if p > 0:
        r["d_case_params"] = eb.check(f"{name} d_case_params", g["d_cp"], dc, dc_b, axes=("sample", "param"))
    print(f"\n[{name}] " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()) + f"  ({time.time() - t0:.1f} s)")


@pytest.mark.parametrize("act,case,depth,p", CONFIGS)
def test_backward_stages_64x64(act, case, depth, p, request):
    b = case if isinstance(case, int) else _batch_for(case)
    _check_all("cavity", act, b, depth, p, f"{request.node.callspec.id} B={b}")


@pytest.mark.parametrize("where,b,depth,p", GRID_CONFIGS)
def test_backward_stages_grid(where, b, depth, p, request):
    _check_all(where, "float32", b, depth, p, request.node.callspec.id)
