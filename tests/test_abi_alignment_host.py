"""The alignment contract of the C ABI, without a GPU.

Every exported entry point checks each caller device pointer against the widest access its kernels make through it --
16 bytes for float4 / uint4 accesses, TMA and bulk copies, 8 for complex64, int64 and four-bf16 (uint2) accesses, 4 or 2
for scalar fp32 / bf16 ones -- and refuses an under-aligned one with status 1 and a message naming the entry point and the
argument, before any device work.  Without the check, a legal PyTorch view that starts 4 bytes into its storage faults the
device.  ALIGN below is that contract written out; it must name every pointer parameter of include/cfdbench_b200.h, so an
entry point added later has to state what it needs.

Each refusal is exercised with every other argument valid-looking (fake, 256-byte aligned device addresses that are never
dereferenced) in a child process that sees no CUDA device: a missing check then shows up as a launch error instead of a
launch on fake addresses.
"""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cfdbench_b200.h")
HOST = "host / struct"   # host memory, a struct of pointers, a host array or the stream handle: not a device operand


def _f(f32, bf16):
    """a requirement that depends on the call's act_dtype / frame_dtype"""
    return {0: f32, 1: bf16}


def _h(*names):
    return {n: HOST for n in names + ("stream",)}


_FWD = _h("w", "ws")                                          # structs of the forward drivers
_TRAIN = _h("w", "saved", "ws")
_BWD = _h("w", "wb", "saved", "grads", "scratch", "ws")
_FRAMES64 = dict(inputs=16, mask=16, case_params=4)          # the 64x64 lift and lift backward read float4
_FRAMES_GRID = dict(inputs=4, mask=4, case_params=4)         # the grid kernels read one float at a time
# (entry point, pointer argument) -> bytes of alignment its kernels need
ALIGN = {
    "fno_pack_spectral_weights": dict(weights1=8, weights2=8, wk=8, stream=HOST),
    "fno_pack_mix_operand": dict(wk=8, wop=4, stream=HOST),
    "fno_pack_mix_operand_from_weights": dict(weights1=8, weights2=8, wop=16, stream=HOST),
    "fno_unpack_spectral_grads": dict(gwk=8, gw1=8, gw2=8, stream=HOST),
    "fno_lift_fwd": dict(_FRAMES64, w=HOST, act_out=16, stream=HOST),
    "fno_spectral_dft_fwd": dict(act_in=16, xm=_f(8, 16), stream=HOST),   # dft_fwd_tc_kernel's launcher needs 16
    "fno_mode_mix": dict(xm=16, wop=16, ym=8, stream=HOST),
    "fno_spectral_inv_kx": dict(ym=8, z=4, stream=HOST),
    "fno_block_out": dict(z=4, act_in=_f(4, 2), w0t=4, bias=4, act_out=_f(4, 2), pre_out=4, pre_in=4, stream=HOST),
    "fno_mode_mix_image": dict(xm=16, wop=16, ym_img=4, stream=HOST),
    "fno_block_fused": dict(ym_img=16, act_in_bf16=16, w0t=4, bias=4, act_out_bf16=16, stream=HOST),
    # bf16 with ws->ym_img and no pre_out: the fused output stage, whose TMA writes act_out
    "fno_block_fwd": dict(w=HOST, act_in=16, act_out=_f(4, 16), pre_out=4, ws=HOST, stream=HOST),
    "fno_project_fwd": dict(act_in=_f(4, 2), mask=4, w=HOST, preds=4, stream=HOST),
    "fno_forward": dict(_FWD, **_FRAMES64, preds=4),
    "fno_rollout": dict(_FWD, **_FRAMES64, preds_seq=16),    # step s + 1's lift reads preds_seq[s]
    "fno_rollout_host": dict(_FWD, inputs_host=HOST, mask_host=HOST, case_params_host=HOST, preds_seq_host=HOST,
                             dev_io=16),
    "fno_forward_train": dict(_TRAIN, **_FRAMES64, preds=4),
    "fno_backward": dict(_BWD, **_FRAMES64, dpreds=4),        # project_bwd_tc_kernel reads dpreds per float
    "fno_backward_inputs": dict(_BWD, **_FRAMES64, dpreds=4, d_inputs=16, d_case_params=4),
    "fno_rollout_forward_train": dict(_TRAIN, **_FRAMES64, preds_seq=16),
    "fno_rollout_backward": dict(_BWD, **_FRAMES64, preds_seq=16, dpreds_seq=16, carry=16, d_inputs=16, d_case_params=4),
    "fno_multistep_metrics": dict(preds_seq=16, label_u=16, mask=16, sums=4, stream=HOST),
    "fno_gather_batch": dict(frames_in=_f(16, 8), frames_out=_f(16, 8), case_table=4, case_ids=4, idx=8, inputs=16,
                             label=16, mask=16, case_params=4, stream=HOST),
    "fno_loss_fwd": dict(preds=16, labels=16, scratch=4, out=4, stream=HOST),
    "fno_loss_bwd": dict(preds=4, labels=4, fwd=4, gout=4, dpreds=4, stream=HOST),
    "fno_adam_step": dict(t=HOST, stream=HOST),
    "fno_train_stage_indices": dict(perm=8, cursor=4, idx_out=8, stream=HOST),
    "fno_adam_step_dev": dict(t=HOST, coef=8, cursor=4, stream=HOST),
    "fno_adam_coefficients": dict(host_out=HOST),
    "fno_train_log_step": dict(loss_out=4, log=4, cursor=4, stream=HOST),
    "fno_grad_norm": dict(tables=HOST, out=4, scratch=8, log=4, cursor=4, stream=HOST),
    "fno_adam_step_ex": dict(t=HOST, clip_coef=4, ema=HOST, stream=HOST),
    "fno_adam_step_dev_ex": dict(t=HOST, coef=8, cursor=4, clip_coef=4, ema=HOST, ema_decay_tab=4, stream=HOST),
    "fno_ema_decays": dict(host_out=HOST),
    "fno_gather_window": dict(frames_in=_f(16, 8), frames_out=_f(16, 8), case_table=4, case_ids=4, idx=8, inputs=16,
                              label=16, mask=16, case_params=4, labels_seq=16, stream=HOST),
    # the losses pick a one-float-at-a-time path for slices that are only 4-byte aligned
    "fno_loss_seq_fwd": dict(preds_seq=4, labels_seq=4, scratch=4, out=4, stream=HOST),
    "fno_loss_seq_bwd": dict(preds_seq=4, labels_seq=4, fwd=4, gout=4, dpreds_seq=4, stream=HOST),
    # the noise kernels take their float4 path only when the frames are 16-byte aligned
    "fno_add_input_noise": dict(inputs=4, mask=4, idx=8, step_base=8, step_offset=4, stream=HOST),
    "fno_add_input_noise_stream": dict(**{"in": 4}, out=4, mask=4, idx=8, step_base=8, step_offset=4, stream=HOST),
    "fno_rollout_noise": dict(_FWD, **_h("noise"), **_FRAMES64, preds_seq=16, fed=16),
    "fno_rollout_forward_train_noise": dict(_TRAIN, **_h("noise"), **_FRAMES64, preds_seq=16, fed=16),
    "fno_rollout_backward_noise": dict(_BWD, **_h("noise"), **_FRAMES64, preds_seq=16, dpreds_seq=16, fed=16, carry=16,
                                       d_inputs=16, d_case_params=4),
    # grid-generic path: frames one float at a time; block_out stages its z rows with float4 copies
    "fno_grid_lift_fwd": dict(_FRAMES_GRID, w=HOST, act_out=4, stream=HOST),
    "fno_grid_spectral_dft_fwd": dict(act_in=4, xm=8, stream=HOST),
    "fno_grid_spectral_inv_kx": dict(ym=8, z=4, stream=HOST),
    "fno_grid_block_out": dict(z=16, act_in=4, w0t=4, bias=4, act_out=4, pre_out=4, pre_in=4, stream=HOST),
    "fno_grid_project_fwd": dict(act_in=4, mask=4, w=HOST, preds=4, stream=HOST),
    "fno_grid_project_bwd": dict(act_in=4, dpreds=4, mask=4, pre=4, w=HOST, dpre_out=4, dz1=4, partials=4, g_fc1_w=4,
                                 g_fc1_b=4, g_fc2_w=4, g_fc2_b=4, stream=HOST),
    "fno_grid_forward": dict(_FWD, **_FRAMES_GRID, preds=4),
    "fno_grid_rollout": dict(_FWD, **_FRAMES_GRID, preds_seq=4),
    "fno_grid_forward_train": dict(_TRAIN, **_FRAMES_GRID, preds=4),
    "fno_grid_backward": dict(_BWD, **_FRAMES_GRID, dpreds=4, d_inputs=4, d_case_params=4),
    "fno_grid_rollout_forward_train": dict(_TRAIN, **_FRAMES_GRID, preds_seq=4),
    "fno_grid_rollout_backward": dict(_BWD, **_FRAMES_GRID, preds_seq=4, dpreds_seq=4, carry=4, d_inputs=4,
                                      d_case_params=4),
    "fno_grid_rollout_noise": dict(_FWD, **_h("noise"), **_FRAMES_GRID, preds_seq=4, fed=4),
    "fno_grid_rollout_forward_train_noise": dict(_TRAIN, **_h("noise"), **_FRAMES_GRID, preds_seq=4, fed=4),
    "fno_grid_rollout_backward_noise": dict(_BWD, **_h("noise"), **_FRAMES_GRID, preds_seq=4, dpreds_seq=4, fed=4,
                                            carry=4, d_inputs=4, d_case_params=4),
    "fno_grid_multistep_metrics": dict(preds_seq=4, label_u=4, mask=4, sums=4, stream=HOST),
    "fno_grid_gather_batch": dict(frames_in=_f(4, 2), frames_out=_f(4, 2), case_table=4, case_ids=4, idx=8, inputs=4,
                                  label=4, mask=4, case_params=4, stream=HOST),
    "fno_grid_gather_window": dict(frames_in=_f(4, 2), frames_out=_f(4, 2), case_table=4, case_ids=4, idx=8, inputs=4,
                                   label=4, mask=4, case_params=4, labels_seq=4, stream=HOST),
    "fno_window_metrics": dict(preds_seq=16, frames_in=_f(16, 8), frames_out=_f(16, 8), starts=8, sums=4, stream=HOST),
    "fno_grid_window_metrics": dict(preds_seq=4, frames_in=_f(4, 2), frames_out=_f(4, 2), starts=8, sums=4, stream=HOST),
    "fno_eval_sums": dict(preds=4, label=4, mask=4, inputs=4, sums=4, stream=HOST),
}


def header_pointer_params():
    """{entry point: [(parameter name, declared type)]} for every pointer parameter declared in the header"""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = {}
    for m in re.finditer(r"\b(?:int|size_t|const char\s*\*)\s+(fno_\w+)\s*\(([^)]*)\)\s*;", src):
        name, params = m.group(1), m.group(2).strip()
        ptrs = []
        for p in (params.split(",") if params and params != "void" else []):
            p = " ".join(p.split())
            if "*" in p:
                ptrs.append((re.findall(r"\w+", p)[-1], p))
        out[name] = ptrs
    return out


def _need(req, dtype):
    return req[dtype] if isinstance(req, dict) else req


# ------------------------------------------------------------------------------------------------ the refusals
_BASE = 1 << 40


class _Fake:
    """distinct, 256-byte aligned device addresses that nothing dereferences"""

    def __init__(self):
        self.n = 0

    def __call__(self):
        self.n += 1
        return _BASE + self.n * 4096


def _structs(lib_mod, fake, grid):
    L = lib_mod
    w = L.FnoWeights(n_layers=4, n_case_params=5)
    for f in ("fc0_w", "fc0_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "gx", "gy"):
        setattr(w, f, fake())
    for a in ("spec_wk", "w0t", "w0_b"):
        arr = getattr(w, a)
        for i in range(L.FNO_MAX_LAYERS):
            arr[i] = fake()
    ws = L.FnoWorkspace()
    ws.act[0], ws.act[1] = fake(), fake()
    ws.xm, ws.ym, ws.z = fake(), fake(), fake()
    ws.ym_img = None if grid else fake()
    saved = L.FnoTrainSaved()
    for i in range(L.FNO_MAX_LAYERS + 1):
        saved.act[i] = fake()
    for i in range(L.FNO_MAX_LAYERS):
        saved.pre[i], saved.xm[i] = fake(), fake()
    wb = L.FnoWeightsBwd()
    for i in range(L.FNO_MAX_LAYERS):
        wb.spec_wkT[i], wb.w0[i] = fake(), fake()
    g = L.FnoGrads()
    for f in ("fc0_w", "fc0_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b"):
        setattr(g, f, fake())
    for a in ("spec_w1", "spec_w2", "w0_w", "w0_b"):
        arr = getattr(g, a)
        for i in range(L.FNO_MAX_LAYERS):
            arr[i] = fake()
    sc = L.FnoBwdScratch()
    sc.d[0], sc.d[1] = fake(), fake()
    sc.dz1, sc.gm, sc.gwk, sc.partials = fake(), fake(), fake(), fake()
    t = L.FnoAdamTensors(count=1)
    t.param[0], t.grad[0], t.exp_avg[0], t.exp_avg_sq[0], t.n[0] = fake(), fake(), fake(), fake(), 4
    nz = L.FnoNoise(std=0.1, seed=1, idx=fake(), step_base=fake(), step_offset=None, k0=0)
    return dict(w=w, ws=ws, saved=saved, wb=wb, g=g, grads=g, sc=sc, scratch_struct=sc, t=t, tables=t, noise=nz)


_INTS = dict(batch=2, steps=2, layer=0, epilogue=0, n_idx=2, n_case_params=5, time_step_size=1, n_frames=16, n_coef=4,
             n_log=4, n_tables=1, stride=2, n_perm=4, noise_stream=1, conj_transpose=0, first_step=1)
_FLOATS = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, s0=1.0, s1=1.0, std=0.1, max_norm=1.0,
               ema_decay=0.5)


def _args(name, decl, lib_mod, fake, dtype, target, offset):
    """the argument list of one call: `target` is offset by `offset` bytes, everything else valid-looking"""
    grid = name.startswith("fno_grid") or name == "fno_eval_sums"
    st = _structs(lib_mod, fake, grid)
    host_keep = []
    params = [" ".join(p.split()) for p in decl.split(",")]
    out = []
    for p in params:
        pname = re.findall(r"\w+", p)[-1]
        if "*" in p:
            kind = ALIGN[name][pname]
            if pname == "stream":
                v = None
            elif pname == "ema":
                v = None                                   # optional host array
            elif kind == HOST and pname.endswith("_host") or pname == "host_out":
                buf = (C.c_float * (2 * 2 * 2 * 4096))()
                host_keep.append(buf)
                v = C.addressof(buf)
            elif kind == HOST:
                key = "scratch_struct" if pname == "scratch" and "fno_bwd_scratch" in p else pname
                v = C.pointer(st[key])
            elif pname == "pre_out" and name == "fno_block_fwd" and target != "pre_out":
                v = None                                   # inference: the fused path for bf16
            elif pname == "step_offset" and target != "step_offset":
                v = None
            else:
                v = fake()
            if pname == target:
                v = v + offset
            out.append(v)
        elif pname in ("act_dtype", "frame_dtype"):
            out.append(dtype)
        elif pname in ("h",):
            out.append(66)
        elif pname in ("w_", "w", "wd"):
            out.append(65)
        elif pname in _INTS:
            out.append(_INTS[pname])
        elif pname in _FLOATS:
            out.append(_FLOATS[pname])
        elif pname == "n":
            out.append(2 if "int n" in p else 4096)
        elif pname in ("step", "seed"):
            out.append(1)
        else:
            raise KeyError(f"{name}: no valid-looking value for {p!r}")
    return out, host_keep


def run_refusals():
    """Call every entry point once per (aligned pointer argument, dtype, under-aligned offset); returns
    [(entry point, argument, dtype, offset, required, status, message)].  Must run where no CUDA device is visible."""
    from cfdbench_b200 import _lib as L
    lib = L.load()
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    decls = {m.group(1): m.group(2) for m in re.finditer(r"\bint\s+(fno_\w+)\s*\(([^)]*)\)\s*;", src)}
    rows = []
    for name, table in ALIGN.items():
        dtypes = (0, 1) if re.search(r"\b(act|frame)_dtype\b", decls[name]) else (0,)
        for target, req in table.items():
            if req == HOST:
                continue
            for dtype in dtypes:
                need = _need(req, dtype)
                for offset in (1, 2, 4, 8):
                    if offset >= need:
                        continue
                    fake = _Fake()
                    args, keep = _args(name, decls[name], L, fake, dtype, target, offset)
                    status = getattr(lib, name)(*args)
                    rows.append((name, target, dtype, offset, need, status, lib.fno_last_error().decode()))
                    del keep
    return rows


_CHILD = """
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_abi_alignment_host as t
print("ROWS" + json.dumps(t.run_refusals()))
"""


def refusals_without_a_device():
    """run_refusals() in a child process that sees no CUDA device, so an unchecked pointer cannot reach a kernel"""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("ROWS")][-1]
    return [tuple(x) for x in json.loads(line[4:])]


def refused(rows):
    """the rows whose call was refused for the right reason: status 1, the entry point and the argument named"""
    return [r for r in rows if r[5] == 1 and r[6] == f"{r[0]}: {r[1]} must be {r[4]}-byte aligned"]


# ------------------------------------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def rows():
    from cfdbench_b200 import build
    build.build()
    return refusals_without_a_device()


def test_every_pointer_parameter_has_an_alignment():
    declared = header_pointer_params()
    missing = [(f, p) for f, ps in declared.items() for p, _ in ps if p not in ALIGN.get(f, {})]
    assert not missing, f"pointer parameters without an entry in ALIGN: {missing}"
    stale = [(f, p) for f, t in ALIGN.items() for p in t if p not in {q for q, _ in declared.get(f, [])}]
    assert not stale, f"ALIGN entries the header does not declare: {stale}"
    for f, t in ALIGN.items():
        for p, req in t.items():
            for need in (req.values() if isinstance(req, dict) else (req,)):
                assert need == HOST or need in (2, 4, 8, 16), (f, p, need)


def test_the_table_matches_the_wrappers_signatures():
    from cfdbench_b200 import _lib
    for f in ALIGN:
        assert f in _lib.SIGNATURES, f


def test_every_under_aligned_pointer_is_refused_before_device_work(rows):
    bad = [r for r in rows if r not in refused(rows)]
    assert not bad, "\n".join(f"{n}({a}) dtype {d} +{o} B (needs {q}): status {s}: {m}" for n, a, d, o, q, s, m in bad)
    # every 16- and 8-byte operand was called at +4 bytes, every bf16 one (2-byte scalar or 8-byte vector) at +2
    called = {(r[0], r[1], r[2], r[3]) for r in rows}
    for f, t in ALIGN.items():
        for p, req in t.items():
            if req == HOST:
                continue
            for dtype, need in (req.items() if isinstance(req, dict) else ((0, req),)):
                if need >= 8:
                    assert (f, p, dtype, 4) in called, (f, p, dtype)
                if dtype == 1:
                    assert (f, p, dtype, 1) in called, (f, p, dtype)


def test_the_16_byte_entry_points_of_the_64x64_path_are_covered(rows):
    """the entry points whose float4 / TMA reads of caller tensors went unchecked before"""
    names = {r[0] for r in refused(rows) if r[4] == 16}
    for f in ("fno_lift_fwd", "fno_forward", "fno_forward_train", "fno_backward", "fno_backward_inputs", "fno_rollout",
              "fno_rollout_forward_train", "fno_rollout_backward", "fno_multistep_metrics", "fno_gather_batch",
              "fno_gather_window", "fno_rollout_noise", "fno_block_fused", "fno_mode_mix", "fno_spectral_dft_fwd",
              "fno_grid_block_out", "fno_window_metrics", "fno_loss_fwd"):
        assert f in names, f


if __name__ == "__main__":
    print(json.dumps(run_refusals()))
