"""dft_fwd_tc_kernel (the bf16-storage forward DFT) against the float64 oracle at batch sizes that hit every unit and
tail case of its mapping: a unit is eight planes of one sample, each warpgroup pipeline walks its units with a stride of
twice the grid, and the grid shrinks to the fewest CTAs that keep the busiest pipeline's unit count.  B = 1, 2 leave
pipelines without units; 33, 67, 255, 257 leave a ragged last round; 256 is the benchmark's batch."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fno_numpy as onp

pytestmark = pytest.mark.gpu

GUARD = 2   # complex64 guard elements on each side of xm: 16 bytes keep the spectrum 16-byte aligned


@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import _lib
    return _lib.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _planes(batch, seed):
    """bf16-exact planes whose scale differs per channel (powers of two), so a plane or row permutation cannot cancel"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((batch, 32, 64, 64)).astype(np.float32)
    x *= (2.0 ** (np.arange(32) % 5 - 2)).astype(np.float32)[None, :, None, None]
    x += np.arange(32, dtype=np.float32)[None, :, None, None] / 8
    return torch.from_numpy(x).to(torch.bfloat16)


def _run(lib, xd, batch, s0=1.0, s1=1.0):
    from cfdbench_b200 import _lib
    n = 288 * batch * 32
    buf = torch.full((n + 2 * GUARD,), complex(-7.25, 3.5), dtype=torch.complex64, device="cuda")
    xm = buf[GUARD:GUARD + n]
    _lib.check(lib.fno_spectral_dft_fwd(xd.data_ptr(), xm.data_ptr(), batch, _lib.ACT_BF16, s0, s1, _stream()), "dft tc")
    torch.cuda.synchronize()
    g = torch.cat([buf[:GUARD], buf[GUARD + n:]]).cpu()
    assert torch.equal(g, torch.full_like(g, complex(-7.25, 3.5))), "write outside xm"
    return xm.view(288, batch, 32).cpu().numpy()


@pytest.mark.parametrize("batch", [1, 2, 33, 67, 255, 256, 257])
def test_dft_fwd_tc_every_unit(lib, batch):
    x = _planes(batch, 100 + batch)
    xd = x.cuda()
    got = _run(lib, xd, batch)
    ref = onp.spectral_modes(x.float().numpy(), 12, 12).reshape(batch, 32, 288).transpose(2, 0, 1)
    err = np.linalg.norm(got - ref, axis=(0, 2)) / np.linalg.norm(ref, axis=(0, 2))   # per sample
    assert err.max() <= 2e-6, (err.argmax(), err.max())
    assert np.abs(got - ref).max() <= 2e-5 * np.abs(ref).max()
    again = _run(lib, xd, batch)
    assert np.array_equal(again.view(np.uint32), got.view(np.uint32)), "not bit-identical over two launches"


def test_dft_fwd_tc_mode_scaling(lib):
    """s0 scales the ky = 0 column, s1 the others"""
    batch = 9
    x = _planes(batch, 7)
    got = _run(lib, x.cuda(), batch, 0.25, 0.5)
    c = np.full(12, 0.5)
    c[0] = 0.25
    ref = (onp.spectral_modes(x.float().numpy(), 12, 12) * c).reshape(batch, 32, 288).transpose(2, 0, 1)
    assert np.linalg.norm(got - ref) / np.linalg.norm(ref) <= 2e-6
