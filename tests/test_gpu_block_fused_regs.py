"""`block_fused_kernel` (fno_block_fused.cu) reads E and the activation row from registers (RS wgmma) and stores its
epilogue with stmatrix.  That moves operand reads only: the products, their order and the accumulation order are those
of the kernel that read both operands from shared memory and stored the tile element by element, so the bf16 output is
the same bit for bit.  The digests below are SHA-256 of the raw bf16 output of that earlier kernel (commit b2b1b7b) on
an H100, recorded with

    python tests/test_gpu_block_fused_regs.py

which prints the digests of the build it runs with.  Inputs are built as tests/test_gpu_fused.py::test_block_fused_kernel
builds them; the rollout is bench.py's headline workload (seeded bf16-storage model, B = 256, 20 steps)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from test_gpu_fused import encode_ym_image  # noqa: E402
from test_gpu_parity import dev, stream  # noqa: E402

pytestmark = pytest.mark.gpu

BATCHES = (1, 3, 80, 257, 1000)
KERNEL_SHA256 = {
    1: "414e925d5b8e5633d678f973c7abe5ea7d563c332468d64b968182f7c0211854",
    3: "95e922cca06e3b961a86bac2a751ff0ad61f595e6b98a86c721ed0a001b42742",
    80: "670e2368c86d83bb5694666d0451d1b36937cb057c9cf19f477cab22ffa311f3",
    257: "f6b3015219b570048292045d7036ffc86c50d7a13ee0263d9a0deaf5ee6decdc",
    1000: "36057f778a68df25049f1158d4a48c8702799874ca52c3c1336fe46221b842f2",
}
ROLLOUT_SHA256 = "0f66324ce32c3d563ad694775d6f0fce5bf0df452948ba4cd3acf6df8542c6eb"


def _lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _block_fused_out(lib, batch):
    from cfdbench_b200 import _lib
    rng = np.random.default_rng(20 + batch)
    ym = (rng.standard_normal((batch, 32, 24, 12)) + 1j * rng.standard_normal((batch, 32, 24, 12))) * 40.0
    ym = ym.astype(np.complex64)
    x = torch.from_numpy(rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)).to(torch.bfloat16)
    w0 = (rng.standard_normal((32, 32)) / 6).astype(np.float32)
    bias = rng.standard_normal(32).astype(np.float32)
    img = torch.from_numpy(encode_ym_image(ym)).cuda()
    xd, w0td, biasd = x.cuda(), dev(w0.T.copy()), dev(bias)
    outs = []
    for fill in (0.0, 3.0):   # two launches into differently pre-filled buffers
        out = torch.full((batch, 32, 64, 64), fill, dtype=torch.bfloat16, device="cuda")
        _lib.check(lib.fno_block_fused(img.data_ptr(), xd.data_ptr(), w0td.data_ptr(), biasd.data_ptr(), out.data_ptr(),
                                       batch, stream()), "block_fused")
        outs.append(out)
    torch.cuda.synchronize()
    return [o.view(torch.int16).cpu().numpy() for o in outs]


def _rollout_preds():
    import bench
    from cfdbench_b200 import synth
    m, _ = bench.build_model("bf16", 5)
    batch = synth.make_batch(1, 256, "cavity", with_label=False)
    inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
    with torch.no_grad():
        seq = m.generate_many(inp, cp, mk, 20)
    torch.cuda.synchronize()
    return torch.stack(seq).cpu().numpy()


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("batch", BATCHES)
def test_block_fused_bits_unchanged(batch):
    a, b = _block_fused_out(_lib(), batch)
    assert np.array_equal(a, b)
    assert _sha(a) == KERNEL_SHA256[batch]


def test_bf16_rollout_bits_unchanged():
    assert _sha(_rollout_preds()) == ROLLOUT_SHA256


if __name__ == "__main__":
    lib = _lib()
    res = {}
    for bt in BATCHES:
        a, b = _block_fused_out(lib, bt)
        res[bt] = _sha(a) if np.array_equal(a, b) else "launches differ"
    print(json.dumps({"kernel": res, "rollout": _sha(_rollout_preds())}))
