"""Device-side evaluation and input batches on every grid the model runs (SURVEY.md 8f.1, 8f.2): the grid-generic
metrics and gather kernels, and `infer_multistep` -- the batched replacement of the reference's `test_multistep.infer`
(src/test_multistep.py:73-177) -- against the per-case loop, a float64 restatement and the reference's own `infer`."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from cfdbench_b200 import synth
from test_data_pipeline import _collate

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.path.join(ROOT, "oracle", "_ref", "src")
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _at(n, offset):
    """A CUDA float32 tensor of n elements that starts `offset` floats into a larger, sentinel-filled buffer, with
    `offset` guard floats on either side."""
    buf = torch.full((n + 2 * offset,), SENTINEL, device="cuda")
    return buf, buf[offset:offset + n]


def _guards_intact(buf, offset):
    return bool((buf[:offset] == SENTINEL).all()) and bool((buf[buf.numel() - offset:] == SENTINEL).all())


def _metrics_ref(preds, label, mask):
    """float64 restatement of get_metrics on the masked u channel and combine_dicts over cases (reference :73-99)."""
    p = preds[:, :, 0].astype(np.float64) * mask
    lab = label.astype(np.float64) * mask
    mse = ((p - lab) ** 2).mean(axis=(2, 3))
    per_case = dict(mse=mse, nmse=mse / (lab ** 2).mean(axis=(2, 3)), mae=np.abs(p - lab).mean(axis=(2, 3)))
    return [{k: float(np.mean(v[s])) for k, v in per_case.items()} for s in range(preds.shape[0])]


def _assert_close(got, ref, rtol):
    assert len(got) == len(ref)
    for s, (g, r) in enumerate(zip(got, ref)):
        assert list(g) == ["mse", "nmse", "mae"]
        for k in g:
            assert abs(g[k] - r[k]) <= rtol * abs(r[k]), (s, k, g[k], r[k])


# ------------------------------------------------------------------------------------------------ metrics kernel
@pytest.mark.parametrize("grid", [(66, 65), (65, 66), (25, 127), (24, 24), (128, 128)])
@pytest.mark.parametrize("sb", [(3, 5), (20, 70)])
def test_grid_metrics_kernel(lib, grid, sb):
    from cfdbench_b200.metrics import multistep_metrics
    (gh, gw), (s, b) = grid, sb
    rng = np.random.default_rng(gh * 1000 + gw + s)
    preds = rng.standard_normal((s, b, 2, gh, gw)).astype(np.float32)
    label = rng.standard_normal((s, b, gh, gw)).astype(np.float32)
    mask = (rng.random((s, b, gh, gw)) > 0.1).astype(np.float32)
    got = multistep_metrics(torch.from_numpy(preds).cuda(), torch.from_numpy(label).cuda(), torch.from_numpy(mask).cuda())
    _assert_close(got, _metrics_ref(preds, label, mask), 2e-6)

    # through the C ABI: inputs one float past an aligned start (label_u / mask planes then start on 4-byte boundaries),
    # sums into a view of a larger buffer whose guard floats must stay untouched; a second launch is bit-identical
    n = s * b * gh * gw
    _, p_d = _at(2 * n, 1)
    _, l_d = _at(n, 1)
    _, m_d = _at(n, 3)
    p_d.copy_(torch.from_numpy(preds.reshape(-1)))
    l_d.copy_(torch.from_numpy(label.reshape(-1)))
    m_d.copy_(torch.from_numpy(mask.reshape(-1)))
    outs = []
    for _ in range(2):
        buf, sums = _at(s * b * 3, 5)
        assert lib.fno_grid_multistep_metrics(p_d.data_ptr(), l_d.data_ptr(), m_d.data_ptr(), sums.data_ptr(), s, b, gh, gw,
                                              _stream()) == 0, lib.fno_last_error()
        torch.cuda.synchronize()
        assert _guards_intact(buf, 5)
        outs.append(sums.clone())
    assert torch.equal(outs[0], outs[1])
    ref = np.stack([((preds[:, :, 0].astype(np.float64) * mask - label * mask) ** 2).sum(axis=(2, 3)),
                    ((label.astype(np.float64) * mask) ** 2).sum(axis=(2, 3)),
                    np.abs(preds[:, :, 0].astype(np.float64) * mask - label * mask).sum(axis=(2, 3))], axis=-1)
    np.testing.assert_allclose(outs[0].view(s, b, 3).cpu().numpy(), ref, rtol=2e-5)


def test_grid_metrics_kernel_agrees_with_64x64_kernel(lib):
    s, b = 4, 9
    rng = np.random.default_rng(64)
    preds = torch.from_numpy(rng.standard_normal((s, b, 2, 64, 64)).astype(np.float32)).cuda()
    label = torch.from_numpy(rng.standard_normal((s, b, 64, 64)).astype(np.float32)).cuda()
    mask = torch.from_numpy((rng.random((s, b, 64, 64)) > 0.1).astype(np.float32)).cuda()
    a = torch.empty(s, b, 3, device="cuda")
    g = torch.empty(s, b, 3, device="cuda")
    assert lib.fno_multistep_metrics(preds.data_ptr(), label.data_ptr(), mask.data_ptr(), a.data_ptr(), s, b, _stream()) == 0
    assert lib.fno_grid_multistep_metrics(preds.data_ptr(), label.data_ptr(), mask.data_ptr(), g.data_ptr(), s, b, 64, 64,
                                          _stream()) == 0
    torch.testing.assert_close(g, a, rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ gather kernel
class _GridAutoDataset(torch.utils.data.Dataset):
    """Attributes and __getitem__ of the reference's auto datasets (TubeFlowAutoDataset / DamFlowAutoDataset hold
    (N, 3, 66, 65) frames, src/dataset/tube.py:228-281) at any grid."""

    def __init__(self, n, gh, gw, n_cases=6, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.inputs = torch.randn(n, 3, gh, gw, generator=g)
        self.inputs[:, 2] = (torch.rand(n, gh, gw, generator=g) > 0.1).float()
        self.labels = torch.randn(n, 3, gh, gw, generator=g)
        self.case_ids = np.sort(np.random.default_rng(seed).integers(0, n_cases, n))
        self.case_params = [dict(vel_in=0.5 + 0.1 * c, density=1.0 + c, viscosity=0.01 * (c + 1), rotated=c % 2,
                                 height=0.1 + 0.02 * c, dx=0.1, width=1.0 - 0.05 * c) for c in range(n_cases)]

    def __len__(self):
        return len(self.inputs)

    def __getitem__(self, idx):
        return self.inputs[idx], self.labels[idx], self.case_params[self.case_ids[idx]]


@pytest.mark.parametrize("grid", [(66, 65), (25, 127), (128, 24)])
@pytest.mark.parametrize("frame_dtype", [torch.float32, torch.bfloat16])
def test_grid_device_batches_equal_collate_fn(lib, grid, frame_dtype):
    from cfdbench_b200 import DeviceFrames, _lib
    gh, gw = grid
    ds = _GridAutoDataset(41, gh, gw, seed=gh + gw)
    frames = DeviceFrames(ds, device="cuda", frame_dtype=frame_dtype)
    g1, g2 = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
    dl = torch.utils.data.DataLoader(ds, batch_size=16, shuffle=True, generator=g1, collate_fn=_collate)
    n_batches = 0
    for got, ref in zip(frames.loader(16, shuffle=True, generator=g2), dl):
        n_batches += 1
        for k in ("inputs", "label", "mask", "case_params"):
            r = ref[k].float()
            if frame_dtype == torch.bfloat16 and k != "case_params":
                r = r.to(torch.bfloat16).float()
            assert got[k].dtype == torch.float32 and got[k].is_contiguous()
            assert tuple(got[k].shape) == tuple(r.shape), k
            assert torch.equal(got[k].cpu(), r), k
    assert n_batches == 3   # 16 + 16 + 9

    # through the C ABI into views of guarded buffers at odd offsets: nothing outside the batch is written
    idx = torch.tensor([40, 0, 17, 17, 3], dtype=torch.int64, device="cuda")
    n, p, hw = idx.numel(), frames.n_case_params, gh * gw
    bufs = [_at(n * 2 * hw, 1), _at(n * 2 * hw, 3), _at(n * hw, 5), _at(n * p, 7)]
    st = lib.fno_grid_gather_batch(frames.frames_in.data_ptr(), frames.frames_out.data_ptr(), frames.case_table.data_ptr(),
                                   frames.case_ids.data_ptr(), idx.data_ptr(), n, p,
                                   _lib.ACT_BF16 if frame_dtype == torch.bfloat16 else _lib.ACT_F32,
                                   *(v.data_ptr() for _, v in bufs), gh, gw, _stream())
    assert st == 0, lib.fno_last_error()
    torch.cuda.synchronize()
    for (buf, _), off in zip(bufs, (1, 3, 5, 7)):
        assert _guards_intact(buf, off)
    ref = frames.batch(idx.cpu())
    for (_, v), k in zip(bufs, ("inputs", "label", "mask", "case_params")):
        assert torch.equal(v.view_as(ref[k]), ref[k]), k


def test_grid_device_batch_feeds_fno2d():
    from cfdbench_b200 import DeviceFrames, Fno2d
    from cfdbench_b200.loss import loss_name_to_fn
    frames = DeviceFrames(_GridAutoDataset(9, 66, 65, seed=1), device="cuda")
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=frames.n_case_params, loss_fn=loss_name_to_fn("nmse"), num_layers=4,
              hidden_dim=32, modes1=12, modes2=12).cuda()
    out = m(**frames.batch([8, 1, 4]))
    assert tuple(out["preds"].shape) == (3, 2, 66, 65) and torch.isfinite(out["loss"]["nmse"])


# ------------------------------------------------------------------------------------------------ infer_multistep
def _model(problem, act_dtype="float32", seed=3):
    from cfdbench_b200 import Fno2d
    from cfdbench_b200.loss import loss_name_to_fn
    p = synth.n_case_params(problem)
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12, act_dtype=act_dtype)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(seed, n_params=p, spectral_gain=20.0).items()})
    return m.cuda()


@pytest.mark.parametrize("problem,act_dtype", [("cavity", "float32"), ("cavity", "bfloat16"), ("cylinder", "float32"),
                                               ("tube", "float32")])
def test_infer_multistep_matches_per_case_loop(problem, act_dtype):
    from cfdbench_b200 import infer_multistep
    steps, max_batch = 6, 16
    feats_np, cps_np = synth.make_split(11, 37, problem, frames=(steps, steps + 3))
    feats = [torch.from_numpy(f).cuda() for f in feats_np]
    cps = [torch.from_numpy(c).cuda() for c in cps_np]
    m = _model(problem, act_dtype)
    with torch.no_grad():
        # the reference's loop: one B = 1 rollout per case (infer_case, src/test_multistep.py:102-132)
        per_case = [torch.stack(m.generate_many(f[0, :-1], c, f[0, -1], steps)) for f, c in zip(feats, cps)]
        # the chunks infer_multistep rolls out: 16 + 16 + 5 cases
        for lo in range(0, len(feats), max_batch):
            chunk = feats[lo:lo + max_batch]
            seq = torch.stack(m.generate_many(torch.stack([f[0, :2] for f in chunk]), torch.stack(cps[lo:lo + max_batch]),
                                              torch.stack([f[0, 2] for f in chunk]), steps))
            for j in range(len(chunk)):   # samples of a batch are computed independently: bit-identical
                assert torch.equal(seq[:, j:j + 1], per_case[lo + j]), (lo + j)
    preds = torch.stack(per_case, dim=1)[:, :, 0].cpu().numpy()    # (S, n, 2, H, W)
    assert np.isfinite(preds).all()
    label = np.stack([f[:steps, 0] for f in feats_np], axis=1)     # prediction s against frame s
    mask = np.stack([f[:steps, 2] for f in feats_np], axis=1)
    got = infer_multistep(m, feats, cps, infer_steps=steps, max_batch=max_batch)
    _assert_close(got, _metrics_ref(preds, label, mask), 2e-6)
    assert infer_multistep(m, feats, cps, infer_steps=steps, max_batch=256) == got
    # host inputs (numpy arrays, CPU tensors) give the same result
    assert infer_multistep(m, feats_np, [torch.from_numpy(c) for c in cps_np], infer_steps=steps, max_batch=256) == got


_REF_INFER = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, {root!r})
from cfdbench_b200 import runner, synth
runner.install({src!r}, stub_missing=True)
import test_multistep
from cfdbench_b200.fno2d import Fno2d          # the class the runner bound to the reference's AutoCfdModel
from cfdbench_b200.loss import loss_name_to_fn
from cfdbench_b200.metrics import infer_multistep
out = {{}}
for problem in ("cavity", "tube"):
    p = synth.n_case_params(problem)
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12)
    m.load_state_dict({{k: torch.from_numpy(v) for k, v in synth.make_state_dict(5, n_params=p, spectral_gain=20.0).items()}})
    m = m.cuda()
    feats, cps = synth.make_split(2, 7, problem, frames=(5, 7))
    feats = [torch.from_numpy(f).cuda() for f in feats]
    cps = [torch.from_numpy(c).cuda() for c in cps]
    ref = test_multistep.infer(m, feats, cps, 5)
    ours = infer_multistep(m, feats, cps, infer_steps=5, max_batch=3)
    out[problem] = dict(ref=[{{k: float(v) for k, v in d.items()}} for d in ref], ours=ours)
print("RESULT " + json.dumps(out))
"""


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF_SRC, "models", "fno")),
                    reason="oracle/_ref/src (installed by __graft_entry__.build()) is not present")
def test_infer_multistep_matches_reference_infer():
    env = {**os.environ, "PYTHONDONTWRITEBYTECODE": "1"}
    r = subprocess.run([sys.executable, "-c", _REF_INFER.format(root=ROOT, src=REF_SRC)], capture_output=True, text=True,
                       env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    out = json.loads(line[len("RESULT "):])
    for problem in ("cavity", "tube"):
        ref, ours = out[problem]["ref"], out[problem]["ours"]
        assert len(ref) == 5
        _assert_close(ours, ref, 1e-5)
