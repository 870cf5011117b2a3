"""The pipelined `block_fused_kernel` (fno_block_fused.cu) beyond what tests/test_gpu_fused.py covers: many wrap-arounds of
the per-warpgroup activation rings, TMA stores that stay inside `out`, and bit-reproducibility.  Same acceptance as
test_block_fused_kernel: within one bf16 ulp (+ the fp32 evaluation error of the pre-activation) of the correctly
rounded float64 result, with < 0.5 % of the elements differing at all."""
import numpy as np
import pytest
import torch

from oracle import fno_numpy as onp

from test_gpu_fused import bf16_ulp, encode_ym_image
from test_gpu_parity import dev, rel, stream

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _inputs(batch, seed):
    rng = np.random.default_rng(seed)
    ym = ((rng.standard_normal((batch, 32, 24, 12)) + 1j * rng.standard_normal((batch, 32, 24, 12))) * 40.0)
    ym = ym.astype(np.complex64)
    x = torch.from_numpy(rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)).to(torch.bfloat16)
    w0 = (rng.standard_normal((32, 32)) / 6).astype(np.float32)
    bias = rng.standard_normal(32).astype(np.float32)
    return ym, x, w0, bias


def _launch(lib, img, x, w0td, biasd, out, batch):
    from cfdbench_b200 import _lib
    _lib.check(lib.fno_block_fused(img.data_ptr(), x.data_ptr(), w0td.data_ptr(), biasd.data_ptr(), out.data_ptr(), batch,
                                   stream()), "block_fused")


def _check_against_oracle(got, ym, x, w0, bias):
    spec = onp.spectral_inverse(ym.astype(np.complex128), 64, 64, 12, 12)
    lin = spec + np.einsum("oi,bihw->bohw", w0.astype(np.float64), x.float().numpy().astype(np.float64))
    lin = lin + bias.astype(np.float64)[None, :, None, None]
    ref = onp.gelu(lin)
    ref16 = torch.from_numpy(ref.astype(np.float32)).to(torch.bfloat16).float().numpy().astype(np.float64)
    assert rel(got, ref) < 3e-3, rel(got, ref)
    diff = np.abs(got - ref16)
    allowed = 1.0001 * bf16_ulp(ref16) + 2e-6 * np.maximum(1.0, np.abs(lin))
    assert np.all(diff <= allowed), float((diff / allowed).max())
    assert (diff > 0).mean() < 5e-3, float((diff > 0).mean())


def test_block_fused_ring_wraparound_large_batch(lib):
    """B = 1000: every CTA runs ~30 units, i.e. ~240 fills per activation ring, so every slot's barrier parity flips
    dozens of times and the image ring hundreds.  Checked on the first and last sample of every sample slot (a CTA's first
    and last unit) plus a seeded random subset."""
    batch = 1000
    ym, x, w0, bias = _inputs(batch, 31)
    img = torch.from_numpy(encode_ym_image(ym)).cuda()
    xd, w0td, biasd = x.cuda(), dev(w0.T.copy()), dev(bias)
    out = torch.zeros(batch, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
    _launch(lib, img, xd, w0td, biasd, out, batch)
    torch.cuda.synchronize()
    slots = min(batch, torch.cuda.get_device_properties(0).multi_processor_count // 4)
    pick = set()
    for s in range(slots):
        pick.add(s)
        pick.add(s + ((batch - 1 - s) // slots) * slots)
    pick |= set(np.random.default_rng(7).choice(batch, 24, replace=False).tolist())
    pick = np.array(sorted(pick))
    got = out[torch.from_numpy(pick).cuda()].float().cpu().numpy().astype(np.float64)
    _check_against_oracle(got, ym[pick], x[torch.from_numpy(pick)], w0, bias)


def test_block_fused_stores_stay_inside_out(lib):
    """x and out are views into larger buffers with two guard samples on each side, filled with a sentinel; a TMA store
    writes whole boxes, so any box outside `out` would show up in the guards."""
    batch, guard = 7, 2
    ym, x, w0, bias = _inputs(batch, 32)
    img = torch.from_numpy(encode_ym_image(ym)).cuda()
    w0td, biasd = dev(w0.T.copy()), dev(bias)
    sentinel = torch.tensor([-12345.0], dtype=torch.bfloat16)
    xbig = torch.full((batch + 2 * guard, 32, 64, 64), float(sentinel), dtype=torch.bfloat16, device="cuda")
    obig = torch.full_like(xbig, float(sentinel))
    xbig[guard:guard + batch] = x.cuda()
    xv, ov = xbig[guard:guard + batch], obig[guard:guard + batch]
    _launch(lib, img, xv, w0td, biasd, ov, batch)
    torch.cuda.synchronize()
    s16 = sentinel.view(torch.int16).item()
    raw = obig.view(torch.int16)
    assert bool((raw[:guard] == s16).all()) and bool((raw[guard + batch:] == s16).all())
    assert bool((xbig.view(torch.int16)[:guard] == s16).all())
    ref = torch.zeros(batch, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
    _launch(lib, img, x.cuda(), w0td, biasd, ref, batch)
    torch.cuda.synchronize()
    assert torch.equal(ov.view(torch.int16), ref.view(torch.int16))
    _check_against_oracle(ov.float().cpu().numpy().astype(np.float64), ym, x, w0, bias)


def test_block_fused_bit_reproducible(lib):
    batch = 80
    ym, x, w0, bias = _inputs(batch, 33)
    img = torch.from_numpy(encode_ym_image(ym)).cuda()
    xd, w0td, biasd = x.cuda(), dev(w0.T.copy()), dev(bias)
    a = torch.zeros(batch, 32, 64, 64, dtype=torch.bfloat16, device="cuda")
    b = torch.full_like(a, 3.0)
    _launch(lib, img, xd, w0td, biasd, a, batch)
    _launch(lib, img, xd, w0td, biasd, b, batch)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
