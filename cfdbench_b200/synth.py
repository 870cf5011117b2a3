"""Deterministic synthetic weights and batches for the FNO hot path.

Everything here is generated with numpy's PCG64 ``default_rng`` (bit-stable across numpy
versions and machines) so that the golden fixtures in ``tests/golden`` only need to store a
seed, not 9.5 MB of spectral weights.  Distributions follow the reference's initialisers:

* spectral weights ``weights1/2``: ``scale * rand(cfloat)`` with ``scale = 1/(C_in*C_out)``
  (reference ``src/models/fno/fno2d.py:30-51``) -> real and imaginary parts U[0,1)/1024;
* 1x1 convs (``nn.Conv2d`` default, kaiming-uniform a=sqrt(5)): weight and bias
  U(-1/sqrt(fan_in), 1/sqrt(fan_in)) (reference ``fno2d.py:104,150-156,175-176``);
* inputs: N(0,1) clipped to +-3 (fields are O(1) after the dataset's BC normalisation,
  reference ``src/dataset/utils.py:24-28``); case params N(0,1) (``dataset/utils.py:8-21``);
* masks: cavity all ones (``src/dataset/cavity.py:31``); cylinder ones with a zeroed disc of
  radius 4..8 px plus zeroed rows 0/63 and column 0 (``src/dataset/cylinder.py:249-275``);
  tube and dam ones on the 66x65 grid with the padded inlet column and the top / bottom wall rows
  zeroed (``src/dataset/tube.py:34-50``, ``src/dataset/dam.py:87-105``).
"""
from __future__ import annotations

import numpy as np

H = 64
W = 64
HIDDEN = 32
MODES = 12
DEPTH = 4
PROJ = 128


def n_case_params(problem: str) -> int:
    """cavity, tube, dam -> 5, cylinder -> 8 (reference src/utils/autoregressive.py:31-37)."""
    return {"cavity": 5, "cylinder": 8, "tube": 5, "dam": 5}[problem]


def grid(problem: str) -> tuple[int, int]:
    """Frame size: 64x64 for cavity and cylinder as stored here; (64 + 2) x (64 + 1) for tube and dam, whose loaders pad
    one inlet column and two wall rows (reference src/utils/autoregressive.py:24-26)."""
    return (H + 2, W + 1) if problem in ("tube", "dam") else (H, W)


def make_state_dict(seed: int, n_params: int = 5, in_chan: int = 2, out_chan: int = 2,
                    hidden: int = HIDDEN, depth: int = DEPTH, modes1: int = MODES,
                    modes2: int = MODES, spectral_gain: float = 1.0) -> dict[str, np.ndarray]:
    """Weights with the reference's ``state_dict`` keys, shapes and dtypes (SURVEY.md 8b).

    ``spectral_gain`` > 1 scales the spectral weights up so that the Fourier branch is not
    negligible next to the 1x1 branch (at the default init it contributes O(1e-2) of the
    block output, which would let a wrong FFT hide behind the tolerance)."""
    rng = np.random.default_rng(seed)

    def conv(co: int, ci: int):
        bound = 1.0 / np.sqrt(ci)
        w = rng.uniform(-bound, bound, size=(co, ci, 1, 1)).astype(np.float32)
        b = rng.uniform(-bound, bound, size=(co,)).astype(np.float32)
        return w, b

    sd: dict[str, np.ndarray] = {}
    sd["fc0.weight"], sd["fc0.bias"] = conv(hidden, in_chan + 3 + n_params)
    scale = spectral_gain / (hidden * hidden)
    for l in range(depth):
        for name in ("weights1", "weights2"):
            re = rng.random(size=(hidden, hidden, modes1, modes2))
            im = rng.random(size=(hidden, hidden, modes1, modes2))
            sd[f"blocks.{l}.conv0.{name}"] = (scale * (re + 1j * im)).astype(np.complex64)
        sd[f"blocks.{l}.w0.weight"], sd[f"blocks.{l}.w0.bias"] = conv(hidden, hidden)
    sd["fc1.weight"], sd["fc1.bias"] = conv(PROJ, hidden)
    sd["fc2.weight"], sd["fc2.bias"] = conv(out_chan, PROJ)
    return sd


def make_mask(rng: np.random.Generator, batch: int, problem: str) -> np.ndarray:
    if problem in ("tube", "dam"):
        gh, gw = grid(problem)
        mask = np.ones((batch, 1, gh, gw), dtype=np.float32)
        mask[:, :, :, 0] = 0.0
        mask[:, :, 0, :] = 0.0
        mask[:, :, gh - 1, :] = 0.0
        return mask
    mask = np.ones((batch, 1, H, W), dtype=np.float32)
    if problem == "cylinder":
        hh, ww = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        for b in range(batch):
            r = rng.uniform(4.0, 8.0)
            ch = rng.uniform(16.0, 48.0)
            cw = rng.uniform(12.0, 40.0)
            mask[b, 0][(hh - ch) ** 2 + (ww - cw) ** 2 <= r * r] = 0.0
            mask[b, 0, 0, :] = 0.0
            mask[b, 0, H - 1, :] = 0.0
            mask[b, 0, :, 0] = 0.0
    return mask


def make_batch(seed: int, batch: int, problem: str = "cavity", in_chan: int = 2,
               with_label: bool = True) -> dict[str, np.ndarray]:
    """One synthetic batch with the keys ``collate_fn`` produces (reference
    src/train_auto.py:53-58): inputs (B,2,H,W), label (B,2,H,W), mask (B,1,H,W),
    case_params (B,p); all float32.  (H, W) = ``grid(problem)``."""
    rng = np.random.default_rng(seed)
    p = n_case_params(problem)
    gh, gw = grid(problem)
    out = {
        "inputs": np.clip(rng.standard_normal((batch, in_chan, gh, gw)), -3, 3).astype(np.float32),
        "case_params": rng.standard_normal((batch, p)).astype(np.float32),
        "mask": make_mask(rng, batch, problem),
    }
    if with_label:
        out["label"] = np.clip(rng.standard_normal((batch, in_chan, gh, gw)), -3, 3).astype(np.float32)
    return out


def make_split(seed: int, n_cases: int, problem: str = "cavity", frames=(20, 20)) -> tuple[list, list]:
    """A synthetic test split in the form `test_multistep.main` hands to `infer` (reference src/test_multistep.py:199-218):
    one (T_c, 3, H, W) float32 array per case (u, v, mask), T_c drawn from frames[0]..frames[1], and one (p,) float32
    case-parameter vector per case.  Each frame's mask is the case's mask with a few extra pixels zeroed, so that the
    per-frame mask of the metrics is distinguishable from the start frame's mask of the rollout."""
    rng = np.random.default_rng(seed)
    gh, gw = grid(problem)
    p = n_case_params(problem)
    feats, cps = [], []
    for _ in range(n_cases):
        t = int(rng.integers(frames[0], frames[1] + 1))
        f = np.empty((t, 3, gh, gw), dtype=np.float32)
        f[:, :2] = np.clip(rng.standard_normal((t, 2, gh, gw)), -3, 3)
        f[:, 2] = make_mask(rng, 1, problem)[0, 0] * (rng.random((t, gh, gw)) > 0.02)
        feats.append(f)
        cps.append(rng.standard_normal(p).astype(np.float32))
    return feats, cps
