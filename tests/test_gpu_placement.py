"""Every public path on the memory a caller hands it, on an H100.

1. Placement: each caller tensor at element offsets 0..3 inside a NaN-filled buffer with a 64-element guard on each side
   (a view that starts 4, 8 or 12 bytes -- 2, 4, 6 for bf16 -- into its storage).  Results are bit-identical to the
   offset-0 call and the guards keep their bits.  The offset-0 calls are also held to float64: MseLoss's five scalars
   and d(preds) element by element, the multistep metric sums, the forward per sample.
2. Poisoned workspaces: every buffer the model caches and every buffer it allocates per call filled with 0xFF bytes (NaN in
   fp32, bf16 and fp64) or with zeros before the same calls, at the batches where the kernels' schedules change: outputs
   and gradients are bit-identical, so no kernel reads an element before writing it, and every output element is written.
3. A non-finite neighbour: NaN / Inf pixels in one sample and a NaN case parameter in another leave every other sample's
   predictions, input gradients and metric sums bit-identical, and surface in the poisoned samples' predictions wherever
   the float64 oracle's are non-finite.

The module first checks, without a device (test_abi_alignment_host), that every entry point refuses an under-aligned
pointer to a 16-byte operand: nothing below can then reach a vector access on a misaligned address.
"""
import numpy as np
import pytest
import torch

from cfdbench_b200 import DeviceFrames, Fno2d, loss_name_to_fn, synth
from cfdbench_b200 import metrics as mt
from cfdbench_b200.loss import MseLoss
from oracle import fno_numpy as onp

from test_abi_alignment_host import ALIGN, HOST, refusals_without_a_device, refused
from test_gpu_backward_bounds import _batch_for
from test_gpu_elementwise_bounds import _fused_batch, _tile_batch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 64
P = 5
# (grid, storage, batch): 64x64 in both storages, the tube / dam grid, and an odd batch on an odd grid, where a K-step
# slice of the rollout's (K, B, 2, H, W) output is only 4-byte aligned
CASES = [((64, 64), "float32", 3), ((64, 64), "bfloat16", 3), ((66, 65), "float32", 3), ((25, 127), "float32", 3)]
CASE_IDS = ["64-f32", "64-bf16", "66x65", "25x127"]


@pytest.fixture(scope="module", autouse=True)
def fault_guard():
    """Fail the module before any launch unless every 16-byte operand refuses a pointer 4 bytes off."""
    ok = {(r[0], r[1], r[2]) for r in refused(refusals_without_a_device()) if r[3] == 4}
    missing = [(f, p, d) for f, t in ALIGN.items() for p, req in t.items() if req != HOST
               for d, need in (req.items() if isinstance(req, dict) else ((0, req),)) if need == 16 and (f, p, d) not in ok]
    if missing:
        pytest.fail(f"under-aligned 16-byte operands that are not refused: {missing}", pytrace=False)


def _model(act, seed=7):
    sd = synth.make_state_dict(seed, n_params=P, spectral_gain=100.0)
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=P, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m, sd


def _batch(grid, b, seed=3):
    rng = np.random.default_rng(seed)
    gh, gw = grid
    mask = np.ones((b, gh, gw), np.float32)
    mask[:, 0, :] = mask[:, gh - 1, :] = mask[:, :, 0] = 0.0
    bt = dict(inputs=np.clip(rng.standard_normal((b, 2, gh, gw)), -3, 3).astype(np.float32) * mask[:, None],
              mask=mask, case_params=rng.standard_normal((b, P)).astype(np.float32),
              label=np.clip(rng.standard_normal((b, 2, gh, gw)), -3, 3).astype(np.float32))
    return {k: torch.from_numpy(v).cuda() for k, v in bt.items()}


class _Placer:
    """Places tensors at an element offset inside NaN-filled buffers with GUARD elements on each side."""

    def __init__(self, off):
        self.off, self.bufs = off, []

    def __call__(self, t):
        t = t.detach()
        n = t.numel()
        buf = torch.full((GUARD + self.off + n + GUARD,), float("nan"), dtype=t.dtype, device=t.device)
        view = buf[GUARD + self.off:GUARD + self.off + n].view(t.shape)
        view.copy_(t)
        assert view.data_ptr() % 16 == (self.off * t.element_size()) % 16
        self.bufs.append((buf, n))
        return view

    def check_guards(self):
        for buf, n in self.bufs:
            bits = buf.view(torch.int16 if buf.element_size() == 2 else torch.int32)
            nan = torch.full((1,), float("nan"), dtype=buf.dtype, device=buf.device).view(bits.dtype)
            lo, hi = bits[:GUARD + self.off], bits[GUARD + self.off + n:]
            assert bool((lo == nan).all()) and bool((hi == nan).all()), "a guard element was written"


def _same(a, b, what):
    if isinstance(a, dict):
        for k in a:
            _same(a[k], b[k], f"{what}.{k}")
        return
    if isinstance(a, (list, tuple)):
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{what}[{i}]")
        return
    if not isinstance(a, torch.Tensor):
        assert a == b or (a != a and b != b), (what, a, b)
        return
    assert a.shape == b.shape and a.dtype == b.dtype, what
    if a.dtype in (torch.float32, torch.bfloat16, torch.complex64):
        a, b = a.reshape(-1).contiguous().view(torch.uint8), b.reshape(-1).contiguous().view(torch.uint8)
    assert torch.equal(a, b), f"{what}: not bit-identical"


def _grads(m):
    return [p.grad.clone() for p in m.parameters()]


def _zero_grads(m):
    for p in m.parameters():
        p.grad = None


def _paths(m, bt, place, steps=3):
    """Every public path fed the caller tensors through `place`; returns their outputs."""
    out = {}
    x, c, mk = place(bt["inputs"]), place(bt["case_params"]), place(bt["mask"])
    with torch.no_grad():
        out["forward"] = m(inputs=x, case_params=c, mask=mk)["preds"].clone()
        out["generate_many"] = torch.stack(m.generate_many(x, c, mk, steps))
    g = torch.from_numpy(np.random.default_rng(11).standard_normal(tuple(bt["inputs"].shape)).astype(np.float32)).cuda()
    # training step with input gradients, the upstream gradient placed too
    _zero_grads(m)
    xi, ci = x.detach().requires_grad_(), c.detach().requires_grad_()
    preds = m(inputs=xi, case_params=ci, mask=mk)["preds"]
    preds.backward(place(g))
    out["train"] = dict(preds=preds.detach().clone(), d_inputs=xi.grad.clone(), d_cp=ci.grad.clone(), params=_grads(m))
    # K-step rollout, forward and backward
    _zero_grads(m)
    xi, ci = x.detach().requires_grad_(), c.detach().requires_grad_()
    seq = m.rollout(xi, ci, mk, steps)
    gs = torch.stack([g * (k + 1) for k in range(steps)])
    seq.backward(place(gs))
    out["rollout"] = dict(seq=seq.detach().clone(), d_inputs=xi.grad.clone(), d_cp=ci.grad.clone(), params=_grads(m))
    # MseLoss forward and backward
    p = place(out["forward"]).detach().requires_grad_()
    lab = place(bt["label"] * bt["mask"][:, None])
    ls = MseLoss(normalize=True)(preds=p, labels=lab)
    sum(ls.values()).backward()
    out["mse"] = dict(loss={k: v.detach().clone() for k, v in ls.items()}, dpreds=p.grad.clone())
    # multistep metrics on the rollout
    s, b = out["generate_many"].shape[:2]
    lu = place(bt["label"][:, 0].expand(s, *bt["label"][:, 0].shape).contiguous())
    mm = place(bt["mask"].expand(s, *bt["mask"].shape).contiguous())
    out["metrics"] = mt.multistep_metrics(place(out["generate_many"]), lu, mm)
    return out


class _Frames:
    """a device-resident split: (N, 3, H, W) frames, labels = frames one step on"""

    def __init__(self, frames, case_params, place):
        self.inputs, self.labels = place(frames[:-1]), place(frames[1:])
        self.case_ids = np.zeros(frames.shape[0] - 1, np.int64)
        self.case_params = [{f"p{j}": float(v) for j, v in enumerate(case_params)}]
        self.time_step_size = 1


@pytest.mark.parametrize("grid, act, b", CASES, ids=CASE_IDS)
def test_placement(grid, act, b):
    m, sd = _model(act)
    bt = _batch(grid, b)
    ref = None
    for off in range(4):
        place = _Placer(off)
        got = _paths(m, bt, place)
        place.check_guards()
        if ref is None:
            ref = got
        else:
            _same(got, ref, f"offset {off}")
    print(f"\n[placement {grid} {act} B={b}] offsets 0-3 bit-identical, guards intact")
    _float64_checks(ref, bt, sd, grid, act)


@pytest.mark.parametrize("frame_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("grid", [(64, 64), (66, 65)])
def test_device_frames_placement(grid, frame_dtype):
    rng = np.random.default_rng(5)
    frames = torch.from_numpy(rng.standard_normal((9, 3, *grid)).astype(np.float32)).cuda()
    frames[:, 2] = (frames[:, 2] > -1).float()
    cp = rng.standard_normal(P).astype(np.float32)
    idx = torch.tensor([5, 0, 3], dtype=torch.int64, device="cuda")   # 3-step windows from 5 and 0 stay in the split
    ref = None
    elt = 2 if frame_dtype == torch.bfloat16 else 4
    for off in range(4):
        place = _Placer(off)
        fr = DeviceFrames(_Frames(frames.to(frame_dtype), cp, place), frame_dtype=frame_dtype)
        got = dict(batch=fr.batch(idx), window=fr.rollout_batch(idx[:2], 3))
        place.check_guards()
        if ref is None:
            ref = got
        else:
            _same(got, ref, f"DeviceFrames {grid} {frame_dtype} offset {off} ({off * elt} bytes)")


# ------------------------------------------------------------------------------------------------ float64 checks
def _gamma(k):
    return k * U / (1 - k * U)


def _float64_checks(ref, bt, sd, grid, act):
    # MseLoss: five scalars against float64; the kernel's longest addition chain per element: its grid-stride float4
    # loop (ceil(n / (4 * 296 * 256)) float4s, 4 terms each), the tail, 5 shuffle levels, 8 warps, 296 block partials
    p = ref["forward"].double().cpu().numpy()
    lab = (bt["label"] * bt["mask"][:, None]).double().cpu().numpy()
    n = p.size
    d = p - lab
    se, sa, sl = (d * d).sum(), np.abs(d).sum(), (lab * lab).sum()
    k = 4 * -(-n // (4 * 296 * 256)) + 3 + 5 + 8 + 296 + 3
    g = _gamma(k)
    want = dict(mse=se / n, rmse=np.sqrt(se / n), mae=sa / n, nmse=se / sl)
    worst = 0.0
    for key, w in want.items():
        bound = (3 * g + 8 * U) * abs(w)
        err = abs(float(ref["mse"]["loss"][key]) - w)
        assert err <= bound, (key, err, bound)
        worst = max(worst, err / bound)
    # d(preds) for the upstream (1, 1, 1, 1), element by element, fed the kernel's own rmse and mean(labels^2):
    # dp = fmaf(kd, d, ka sgn(d)), kd = (2 + 1 / rmse + 2 / ml2) / n, ka = 1 / n -- a handful of roundings per element
    rmse = float(ref["mse"]["loss"]["rmse"])
    ml2 = float(ref["mse"]["loss"]["mse"]) / float(ref["mse"]["loss"]["nmse"])   # the kernel's mean(labels^2), +2 roundings
    kd = (2.0 + 1.0 / rmse + 2.0 / ml2) / n
    dp_ref = kd * d + np.sign(d) / n
    # kd: 1/n, 1/rmse, 2/ml2 (ml2 recovered: 2 more), three adds, one multiply; d and the fmaf: one each
    bound = 16 * U * (np.abs(kd * d) + 1.0 / n)
    err = np.abs(ref["mse"]["dpreds"].double().cpu().numpy() - dp_ref)
    assert (err <= bound).all(), float((err / bound).max())
    worst_dp = float((err / bound).max())
    # multistep metric sums: per plane, per thread ceil(hw / 256) fmaf / adds, 5 shuffle levels, 8 warps
    seq = ref["generate_many"].double().cpu().numpy()
    s, b, _, gh, gw = seq.shape
    m = bt["mask"].double().cpu().numpy()
    lu = bt["label"][:, 0].double().cpu().numpy()
    hw = gh * gw
    k = -(-hw // 256) * (4 if (gh, gw) == (64, 64) else 1) + 5 + 8 + 2
    got = mt.multistep_metrics(ref["generate_many"], bt["label"][:, 0].expand(s, b, gh, gw), bt["mask"].expand(s, b, gh, gw))
    worst_m = 0.0
    for st in range(s):
        pp, ll = seq[st, :, 0] * m, lu * m
        dd = pp - ll
        e, l2, a = (dd * dd).sum((1, 2)), (ll * ll).sum((1, 2)), np.abs(dd).sum((1, 2))
        mse, mae = e / hw, a / hw
        for key, w, rel in (("mse", mse.mean(), 3 * _gamma(k)), ("mae", mae.mean(), 2 * _gamma(k)),
                            ("nmse", (e / l2).mean(), 5 * _gamma(k))):
            bound = (rel + 8 * U) * abs(w)
            err = abs(got[st][key] - w)
            assert err <= bound, (st, key, err, bound)
            worst_m = max(worst_m, err / bound)
    line = f"[float64 {grid} {act}] MseLoss scalars {worst:.3f}, dpreds {worst_dp:.3f}, metric sums {worst_m:.3f} of the bound"
    # the forward, per sample, against the float64 oracle (64x64 fp32: the parity bar of test_gpu_parity.py)
    # the forward, per sample, against the float64 oracle: fp32 storage at the smoke test's 1e-5, bf16 storage against the
    # bf16-boundary oracle (hidden activations rounded to bf16) at its 3e-3
    bn = {k: v.cpu().numpy() for k, v in bt.items()}
    bf = act == "bfloat16"
    fw = onp.fno_forward(sd, bn["inputs"], bn["case_params"], bn["mask"][:, None],
                         round_fn=onp.bf16_round if bf else None)["preds"]
    per = [onp.rel_l2(p[i:i + 1], fw[i:i + 1]) for i in range(p.shape[0])]
    assert max(per) < (3e-3 if bf else 1e-5), per
    line += f", forward per-sample rel-L2 max {max(per):.2e}"
    print(line)


# ------------------------------------------------------------------------------------------------ poisoned workspaces
_EXCLUDED = {
    "_packed": "packed weights and coordinate tables: rebuilt when the weights change, not workspace",
    "sw": "graph-owned copies of the packed weights and coordinate tables",
}
# the loss's partial-sum table (_NativeLoss._scratch) is documented as zero between calls (the kernel leaves it zeroed);
# no optimizer takes part here


def _cached_tensors(obj, seen, out, path="m"):
    if isinstance(obj, torch.Tensor):
        if obj.is_cuda and id(obj) not in seen:
            seen.add(id(obj))
            out.append((path, obj))
        return
    if isinstance(obj, dict):
        for k, v in obj.items():
            if k in _EXCLUDED:
                continue
            _cached_tensors(v, seen, out, f"{path}[{k!r}]")
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _cached_tensors(v, seen, out, f"{path}[{i}]")


def _poison(m, byte):
    """Fill every CUDA tensor the model caches with `byte`; returns the count."""
    out, packed = [], []
    _cached_tensors(m._packed, set(), packed)   # the graphs keep the packing they captured: skip it wherever it shows
    seen = {id(p) for p in m.parameters()} | {id(t) for _, t in packed}
    for name in ("_ws_cache", "_graphs", "_train_graphs"):
        _cached_tensors(getattr(m, name), seen, out, name)
    for path, t in out:
        assert t.is_contiguous(), path
        t.view(-1).view(torch.uint8).fill_(byte)
    torch.cuda.synchronize()
    return len(out)


class _PoisonFresh:
    """While active, every CUDA tensor torch.empty / torch.empty_like returns has its storage filled with `byte` first:
    the buffers the model allocates per call (the single-step saved set, the backward scratch d0 / d1 / dz1 / gm / gwk /
    partials, the flat gradient buffer, the predictions, d_inputs, d_case_params) start poisoned whatever the caching
    allocator hands back.  Nothing is filled while a stream is being captured into a graph."""

    def __init__(self, byte):
        self.byte, self.n = byte, 0

    def _fill(self, t):
        if t.is_cuda and t.numel() > 0 and not torch.cuda.is_current_stream_capturing():
            t.untyped_storage().fill_(self.byte)
            self.n += 1
        return t

    def __enter__(self):
        self._empty, self._empty_like = torch.empty, torch.empty_like
        torch.empty = lambda *a, **k: self._fill(self._empty(*a, **k))
        torch.empty_like = lambda *a, **k: self._fill(self._empty_like(*a, **k))
        return self

    def __exit__(self, *exc):
        torch.empty, torch.empty_like = self._empty, self._empty_like


def _workload(m, bt, steps=2):
    out = {}
    x, c, mk = bt["inputs"], bt["case_params"], bt["mask"]
    with torch.no_grad():
        out["forward"] = m(inputs=x, case_params=c, mask=mk)["preds"].clone()
        out["generate_many"] = torch.stack(m.generate_many(x, c, mk, steps))
    g = bt["label"]
    _zero_grads(m)
    xi, ci = x.clone().requires_grad_(), c.clone().requires_grad_()
    preds = m(inputs=xi, case_params=ci, mask=mk)["preds"]
    preds.backward(g)
    out["train"] = dict(preds=preds.detach().clone(), d_inputs=xi.grad.clone(), d_cp=ci.grad.clone(), params=_grads(m))
    _zero_grads(m)
    xi, ci = x.clone().requires_grad_(), c.clone().requires_grad_()
    seq = m.rollout(xi, ci, mk, steps)
    seq.backward(torch.stack([g] * steps))
    out["rollout"] = dict(seq=seq.detach().clone(), d_inputs=xi.grad.clone(), d_cp=ci.grad.clone(), params=_grads(m))
    torch.cuda.synchronize()
    return out


def _finite(o, what):
    if isinstance(o, dict):
        for k, v in o.items():
            _finite(v, f"{what}.{k}")
    elif isinstance(o, (list, tuple)):
        for i, v in enumerate(o):
            _finite(v, f"{what}[{i}]")
    else:
        assert bool(torch.isfinite(o).all()), f"{what}: an element was not written (still NaN from the poison)"


POISON_CASES = [("float32", "ragged tile", lambda: _tile_batch("ragged")),
                ("bfloat16", "fused wrap", lambda: _fused_batch("first_wrap")),
                ("bfloat16", "fused ragged", lambda: _fused_batch("ragged")),
                ("float32", "bwd chunks", lambda: _batch_for("chunks")),
                ("bfloat16", "bwd co_wrap", lambda: _batch_for("co_wrap")),
                ("float32", "one", lambda: 1)]


@pytest.mark.parametrize("act, case, batch", POISON_CASES, ids=[f"{a}-{c}" for a, c, _ in POISON_CASES])
def test_poisoned_workspaces_64x64(act, case, batch):
    _poisoned((64, 64), act, batch())


@pytest.mark.parametrize("b", [3, 33])
def test_poisoned_workspaces_grid(b):
    _poisoned((66, 65), "float32", b)


def _poisoned(grid, act, b):
    m, _ = _model(act)
    bt = _batch(grid, b)
    _workload(m, bt)                     # builds every cache and graph the paths use
    runs = {}
    for byte in (0x00, 0xFF):
        n_cached = _poison(m, byte)
        with _PoisonFresh(byte) as fresh:
            runs[byte] = _workload(m, bt)
        assert n_cached > 0 and fresh.n > 0
    _finite(runs[0xFF], "0xFF")
    _same(runs[0xFF], runs[0x00], f"{grid} {act} B={b}: 0xFF vs zero workspaces")
    print(f"\n[poison {grid} {act} B={b}] {n_cached} cached buffers and {fresh.n} per-call allocations poisoned; outputs "
          f"and gradients bit-identical to zero-filled workspaces")


# ------------------------------------------------------------------------------------------------ non-finite neighbours
@pytest.mark.parametrize("grid, act", [((64, 64), "float32"), ((64, 64), "bfloat16"), ((66, 65), "float32")],
                         ids=["64-f32", "64-bf16", "66x65"])
def test_non_finite_neighbour(grid, act):
    b = _tile_batch("ragged") if grid == (64, 64) else 33
    m, _ = _model(act)
    clean = _batch(grid, b)
    bad, hit = _poisoned_batch(grid, b)
    keep = torch.tensor([i for i in range(b) if i not in hit], device="cuda")

    def run(bt):
        o = _workload(m, bt)
        s = torch.empty(2, b, 3, device="cuda")
        seq = o["rollout"]["seq"]
        mt._launch_metrics(seq.contiguous(), bt["label"][:, 0].expand(2, b, *grid).contiguous(),
                           bt["mask"].expand(2, b, *grid).contiguous(), s)
        o["sums"] = s
        return o
    a, z = run(clean), run(bad)
    sel = lambda t, dim=0: t.index_select(dim, keep)   # noqa: E731
    _same(sel(z["forward"]), sel(a["forward"]), "forward")
    _same(sel(z["generate_many"], 1), sel(a["generate_many"], 1), "generate_many")
    _same(sel(z["rollout"]["seq"], 1), sel(a["rollout"]["seq"], 1), "rollout")
    _same(sel(z["sums"], 1), sel(a["sums"], 1), "metric sums")
    for path in ("train", "rollout"):
        _same(sel(z[path]["d_inputs"]), sel(a[path]["d_inputs"]), f"{path} d_inputs")
        _same(sel(z[path]["d_cp"]), sel(a[path]["d_cp"]), f"{path} d_case_params")
        assert not all(bool(torch.isfinite(g).all()) for g in z[path]["params"]), f"{path}: the NaN was swallowed"
    print(f"\n[non-finite {grid} {act} B={b}] samples {hit} poisoned; every other sample bit-identical")


def _poisoned_batch(grid, b):
    bad = _batch(grid, b)
    bad["inputs"][1, 0, 9, 17] = float("nan")
    bad["inputs"][1, 1, min(30, grid[0] - 2), min(40, grid[1] - 2)] = float("inf")
    bad["case_params"][b - 2, 0] = float("nan")
    return bad, [1, b - 2]


# A NaN or Inf in a sample has to reach that sample's predictions on every route.  The DFT spreads one non-finite pixel
# over all of a plane's modes, so from the first Fourier layer on the oracle's poisoned samples are non-finite
# throughout; every later stage -- the 3xTF32 / bf16 tensor-core stages of the 64 x 64 path included, whose operand split
# tc::round_tf32 keeps NaN a NaN -- must carry that through, in one forward, in generate_many's feedback and in
# Fno2d.rollout.  test_gpu_non_finite checks the same stage by stage, element by element.
@pytest.mark.parametrize("grid, act", [((64, 64), "float32"), ((64, 64), "bfloat16"), ((66, 65), "float32"),
                                       ((25, 127), "float32")], ids=["64-f32", "64-bf16", "66x65", "25x127"])
def test_non_finite_sample_surfaces(grid, act):
    """The poisoned samples' predictions are non-finite wherever the float64 oracle's are: forward, generate_many and
    Fno2d.rollout, two steps."""
    b = _tile_batch("ragged") if grid == (64, 64) else 33
    steps = 2
    m, sd = _model(act)
    bad, hit = _poisoned_batch(grid, b)
    x, c, mk = bad["inputs"], bad["case_params"], bad["mask"]
    with torch.no_grad():
        got = {"forward": m(inputs=x, case_params=c, mask=mk)["preds"][hit][None],
               "generate_many": torch.stack(m.generate_many(x, c, mk, steps))[:, hit],
               "rollout": m.rollout(x, c, mk, steps)[:, hit]}
    bn = {k: v[hit].cpu().numpy() for k, v in bad.items()}
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.stack(onp.rollout(sd, bn["inputs"], bn["case_params"], bn["mask"], steps))
    if np.isfinite(r[0]).all():
        pytest.fail("the oracle's predictions of the poisoned samples are finite: the set-up is wrong")
    for what, t in got.items():
        z = t.float().cpu().numpy()
        assert (~np.isfinite(z))[~np.isfinite(r[:len(z)])].all(), \
            f"{what}: an element the oracle makes non-finite came out finite"



# ------------------------------------------------------------------------------------------------ scalar paths, called directly
def _stream():
    import ctypes as C
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _loss_rows(p, lab, n, k_chain):
    """float64 (mse, rmse, mae, nmse, mean(labels^2)) of one step and the relative bound of each"""
    d = p - lab
    se, sa, sl = (d * d).sum(), np.abs(d).sum(), (lab * lab).sum()
    g = _gamma(k_chain)
    want = np.array([se / n, np.sqrt(se / n), sa / n, se / sl, sl / n])
    rel = np.array([g, g / 2, g, 2 * g, g]) + 8 * U
    return want, rel


@pytest.mark.parametrize("grid", [(64, 64), (66, 65), (25, 127)])
def test_scalar_path_entry_points_on_4_byte_aligned_pointers(grid):
    """fno_eval_sums, fno_loss_seq_fwd / _bwd, fno_loss_bwd, fno_add_input_noise and the grid forward's frames take
    4-byte aligned pointers: called directly at element offsets 0..3 inside NaN guards, they give the offset-0 bits,
    leave the guards alone and stay within their float64 bounds.  On 64x64 the forward refuses them instead."""
    from cfdbench_b200 import _lib
    lib = _lib.load()
    gh, gw = grid
    b, steps, hw = 3, 2, gh * gw
    bt = _batch(grid, b, seed=9)
    rng = np.random.default_rng(4)
    preds = torch.from_numpy(rng.standard_normal((steps, b, 2, gh, gw)).astype(np.float32)).cuda()
    labels = torch.from_numpy(rng.standard_normal((steps, b, 2, gh, gw)).astype(np.float32)).cuda()
    n = b * 2 * hw
    k_chain = 4 * -(-n // (4 * 296 * 256)) + 3 + 5 + 8 + 296 + 3
    ref, worst = None, 0.0
    for off in range(4):
        place = _Placer(off)
        got = {}
        # eval sums: sums [B][6]
        sums = place(torch.zeros(b, 6, device="cuda"))
        pm = preds[0] * bt["mask"][:, None]
        _lib.check(lib.fno_eval_sums(place(pm).data_ptr(), place(bt["label"]).data_ptr(), place(bt["mask"]).data_ptr(),
                                     place(bt["inputs"]).data_ptr(), sums.data_ptr(), b, gh, gw, _stream()),
                   "fno_eval_sums")
        got["eval"] = sums.clone()
        # K-step loss forward / backward and the one-step backward
        ps, ls = place(preds), place(labels)
        scratch = torch.zeros(lib.fno_loss_seq_scratch_bytes(steps), dtype=torch.uint8, device="cuda")
        out = place(torch.zeros(steps + 1, 5, device="cuda"))
        _lib.check(lib.fno_loss_seq_fwd(ps.data_ptr(), ls.data_ptr(), n, steps, scratch.data_ptr(), out.data_ptr(),
                                        _stream()), "fno_loss_seq_fwd")
        gout = place(torch.ones(4, device="cuda"))
        dseq = place(torch.zeros(steps, b, 2, gh, gw, device="cuda"))
        _lib.check(lib.fno_loss_seq_bwd(ps.data_ptr(), ls.data_ptr(), out.data_ptr(), gout.data_ptr(), dseq.data_ptr(), n,
                                        steps, _stream()), "fno_loss_seq_bwd")
        d1 = place(torch.zeros(b, 2, gh, gw, device="cuda"))
        _lib.check(lib.fno_loss_bwd(ps.data_ptr(), ls.data_ptr(), out.data_ptr(), gout.data_ptr(), d1.data_ptr(), n,
                                    _stream()), "fno_loss_bwd")
        got.update(loss=out.clone(), dseq=dseq.clone(), d1=d1.clone())
        # the noise kernel: a vector path only for 16-byte aligned 64x64 frames
        x = place(bt["inputs"])
        idx = torch.arange(b, dtype=torch.int64, device="cuda")
        step = torch.full((1,), 7, dtype=torch.int64, device="cuda")
        _lib.check(lib.fno_add_input_noise(x.data_ptr(), place(bt["mask"]).data_ptr(), idx.data_ptr(), b, gh, gw, 0.1, 5,
                                           step.data_ptr(), None, _stream()), "fno_add_input_noise")
        got["noise"] = x.clone()
        torch.cuda.synchronize()
        place.check_guards()
        if ref is None:
            ref = got
        else:
            _same(got, ref, f"{grid} offset {off}")
    # float64: eval sums
    p64, l64, m64 = (t.double().cpu().numpy() for t in (preds[0] * bt["mask"][:, None], bt["label"], bt["mask"]))
    x64 = bt["inputs"].double().cpu().numpy()
    lm = l64 * m64[:, None]
    terms = [(p64 - lm) ** 2, np.abs(p64 - lm), lm ** 2]
    want = np.stack([t.sum((1, 2, 3)) for t in terms] +
                    [((x64[:, 0] - l64[:, 0]) ** 2).sum((1, 2)), np.abs(x64[:, 0] - l64[:, 0]).sum((1, 2)),
                     (l64[:, 0] ** 2).sum((1, 2))], 1)
    bound = (_gamma(2 * hw + 3)) * np.abs(want) + 1e-30
    err = np.abs(ref["eval"].double().cpu().numpy() - want)
    assert (err <= bound).all(), float((err / bound).max())
    worst = max(worst, float((err / bound).max()))
    # float64: the K-step loss rows and their mean
    pp, lab = preds.double().cpu().numpy(), labels.double().cpu().numpy()
    rows = ref["loss"].double().cpu().numpy()
    for k in range(steps):
        w, rel = _loss_rows(pp[k], lab[k], n, k_chain)
        e = np.abs(rows[k] - w)
        assert (e <= rel * np.abs(w)).all(), (k, e / (rel * np.abs(w)))
        worst = max(worst, float((e / (rel * np.abs(w))).max()))
    assert np.array_equal(rows[steps].astype(np.float32), ((rows[0] + rows[1]).astype(np.float32) *
                                                           np.float32(1 / steps)).astype(np.float32))
    # float64: d(preds) element by element for gout * (1/steps), fed the kernel's own rmse and mean(labels^2)
    for k in range(steps):
        gk = 1.0 / steps
        kd = gk * (2.0 + 1.0 / rows[k, 1] + 2.0 / rows[k, 4]) / n
        d = pp[k] - lab[k]
        dp = kd * d + gk * np.sign(d) / n
        e = np.abs(ref["dseq"][k].double().cpu().numpy() - dp)
        bound = 16 * U * (np.abs(kd * d) + gk / n)
        assert (e <= bound).all(), float((e / bound).max())
        worst = max(worst, float((e / bound).max()))
    # fno_loss_bwd with the aggregate row's gout read as one step's: the same formula with gk = 1 on step 0
    kd = (2.0 + 1.0 / rows[0, 1] + 2.0 / rows[0, 4]) / n
    d = pp[0] - lab[0]
    e = np.abs(ref["d1"].double().cpu().numpy() - (kd * d + np.sign(d) / n))
    bound = 16 * U * (np.abs(kd * d) + 1.0 / n)
    assert (e <= bound).all(), float((e / bound).max())
    # the grid forward's frames directly at offsets 1..3 (the module would copy them); 64x64 refuses them
    m, sd = _model("float32")
    base = m._native_forward(bt["inputs"], bt["mask"][:, None].contiguous(), bt["case_params"])
    for off in (1, 2, 3):
        place = _Placer(off)
        args = (place(bt["inputs"]), place(bt["mask"][:, None].contiguous()), place(bt["case_params"]))
        if grid == (64, 64):
            with pytest.raises(_lib.FnoNativeError, match="must be 16-byte aligned"):
                m._native_forward(*args)
        else:
            _same(m._native_forward(*args), base, f"grid forward offset {off}")
            place.check_guards()
    print(f"\n[scalar paths {grid}] offsets 0-3 bit-identical, guards intact; eval sums, loss rows and d(preds) at most "
          f"{worst:.3f} of their float64 bounds")
