"""Training noise and pushforward training (`train_auto(input_noise_std=..., rollout_grad_steps=...)`) without a GPU:
a numpy restatement of the noise kernel's Philox4x32-10 against Random123's known-answer vectors, the float64
Box-Muller built on it, the new entry point's declaration and argument checks, and the refusals of `train_auto` and
`DeviceFrames.batch` / `rollout_batch`, all of which run before any device work.

`noise_reference` is the host restatement the GPU tests compare the kernel against."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cfdbench_b200
from cfdbench_b200 import DeviceFrames, _lib, train_auto
from test_train_auto_host import _cpu_model, _Split
from test_train_rollout_host import _TimedSplit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC'11; Random123's philox4x32 with 10 rounds), vectorised: counter (..., 4) and
    key (..., 2) arrays of uint32 words -> (..., 4) uint32."""
    c = [np.asarray(counter, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = (np.asarray(key, dtype=np.uint64)[..., i] for i in range(2))
    mask = np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r > 0:
            k0, k1 = (k0 + np.uint64(_W0)) & mask, (k1 + np.uint64(_W1)) & mask
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
    return np.stack(c, axis=-1).astype(np.uint32)


def uniform_f32(x):
    """curand's uniform in (0, 1], as the kernel forms it in float32: float(x) * 2^-32 + 2^-33."""
    return np.asarray(x, dtype=np.uint32).astype(np.float32) * np.float32(2.0 ** -32) + np.float32(2.0 ** -33)


def noise_reference(seed: int, step: int, j: int, n_el: int) -> np.ndarray:
    """The float64 normals z[0..n_el) of sample j at (seed, step): Box-Muller on the kernel's float32 uniforms of
    Philox4x32-10(counter = (q, j, step_lo, step_hi), key = (seed_lo, seed_hi)), four normals per quad q."""
    nq = (n_el + 3) // 4
    ctr = np.zeros((nq, 4), np.uint64)
    ctr[:, 0] = np.arange(nq)
    ctr[:, 1] = j & 0xFFFFFFFF
    ctr[:, 2] = step & 0xFFFFFFFF
    ctr[:, 3] = step >> 32
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint64)
    u = uniform_f32(philox4x32_10(ctr, key)).astype(np.float64)
    r0, t0 = np.sqrt(-2.0 * np.log(u[:, 0])), 2.0 * u[:, 1]
    r1, t1 = np.sqrt(-2.0 * np.log(u[:, 2])), 2.0 * u[:, 3]
    z = np.stack([r0 * np.cos(np.pi * t0), r0 * np.sin(np.pi * t0), r1 * np.cos(np.pi * t1), r1 * np.sin(np.pi * t1)], 1)
    return z.reshape(-1)[:n_el]


# ------------------------------------------------------------------------------------------------ the RNG
@pytest.mark.parametrize("counter,key,expect", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(counter, key, expect):
    got = philox4x32_10(np.array([counter], np.uint64), np.array([key], np.uint64))[0]
    assert [int(v) for v in got] == list(expect)


def test_uniform_lies_in_the_half_open_unit_interval():
    u = uniform_f32(np.array([0, 1, 2 ** 31, 2 ** 32 - 129, 2 ** 32 - 1], np.uint64))
    assert u.dtype == np.float32
    assert u[0] == np.float32(2.0 ** -33) and u[-1] == np.float32(1.0) and np.all(u > 0) and np.all(u <= 1)


def test_box_muller_reference():
    z = noise_reference(seed=2 ** 40 + 5, step=7, j=3, n_el=2 * 25 * 127)   # an odd H*W: the last quad is partial
    assert z.shape == (2 * 25 * 127,) and np.all(np.isfinite(z))
    assert abs(z.mean()) < 6 / np.sqrt(z.size) and abs(z.var() - 1) < 6 * np.sqrt(2 / z.size)
    # the quad structure: element 4q + r is component r of quad q, whatever the frame's length
    assert np.array_equal(noise_reference(2 ** 40 + 5, 7, 3, 64)[:8], z[:8])
    # the counter words: each of seed (both halves), step (both halves) and j changes the stream
    for other in ((2 ** 40 + 4, 7, 3), (5, 7, 3), (2 ** 40 + 5, 7 + 2 ** 32, 3), (2 ** 40 + 5, 8, 3), (2 ** 40 + 5, 7, 4)):
        assert not np.any(noise_reference(*other, n_el=64) == z[:64]), other
    # one quad by hand
    x = philox4x32_10(np.array([[1, 3, 7, 0]], np.uint64), np.array([[5, 256]], np.uint64))[0]
    u = uniform_f32(x).astype(np.float64)
    r = np.sqrt(-2 * np.log(u[0]))
    assert np.isclose(z[4], r * np.cos(2 * np.pi * u[1]), rtol=1e-12, atol=1e-12)
    assert np.isclose(z[5], r * np.sin(2 * np.pi * u[1]), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    from cfdbench_b200 import build
    build.build()
    return _lib.load()


def test_noise_entry_point_is_declared_and_exported(lib):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cfdbench_b200.h")).read(), flags=re.S)
    assert re.search(r"\bint\s+fno_add_input_noise\s*\(", hdr)
    assert hasattr(C.CDLL(_lib.LIB_PATH), "fno_add_input_noise")
    assert "fno_add_input_noise" in _lib.SIGNATURES
    assert lib.fno_version() == 4


def test_noise_entry_point_rejects_bad_arguments(lib):
    one = C.c_void_p(16)   # never dereferenced: every call below fails its argument checks first

    def call(x=one, m=one, idx=one, n=4, h=64, w=64, std=1.0, seed=1, base=one, off=one):
        return lib.fno_add_input_noise(x, m, idx, n, h, w, std, seed, base, off, C.c_void_p(0))
    for kw in (dict(x=None), dict(m=None), dict(idx=None), dict(base=None), dict(n=0), dict(n=-3), dict(std=-1.0),
               dict(std=-1e-30), dict(std=float("nan")), dict(std=float("inf")), dict(std=float("-inf")),
               dict(h=66, w=65, x=None), dict(h=25, w=127, std=float("nan"))):
        assert call(**kw) == 1, kw
        assert b"fno_add_input_noise" in lib.fno_last_error()
    for h, w in ((23, 64), (64, 129), (0, 0), (128, 23)):
        assert call(h=h, w=w) == 3, (h, w)
        assert call(h=h, w=w, x=None, std=-1.0) == 3   # the grid check comes first
        assert b"fno_add_input_noise" in lib.fno_last_error()


# ------------------------------------------------------------------------------------------------ Python refusals
BAD_STD = (-1.0, -1e-30, float("nan"), float("inf"), -float("inf"), 1e39, "0.1", None, True, 1j)
BAD_SEED = (-1, 2 ** 64, 1.0, "3", None, True)


def test_device_frames_reject_bad_noise_arguments():
    fr = DeviceFrames.__new__(DeviceFrames)   # no device: every call below fails its argument checks first
    for fn in (lambda **kw: fr.batch([0], **kw), lambda **kw: fr.rollout_batch([0], 2, **kw)):
        for std in BAD_STD:
            with pytest.raises(ValueError, match="noise_std must be a real number >= 0"):
                fn(noise_std=std)
        for seed in BAD_SEED:
            with pytest.raises(ValueError, match=r"noise_seed must be an int in \[0, 2\^64\)"):
                fn(noise_std=0.1, noise_seed=seed)
        for step in (-1, 2 ** 63, 2.0, None, False):
            with pytest.raises(ValueError, match=r"noise_step must be an int in \[0, 2\^63\)"):
                fn(noise_std=0.1, noise_step=step)


def test_train_auto_rejects_bad_noise_and_pushforward_arguments(tmp_path):
    out = tmp_path / "out"
    tr, dv = _TimedSplit(12), _Split(3)
    m = _cpu_model()
    for std in BAD_STD:
        with pytest.raises(ValueError, match="input_noise_std must be a real number >= 0"):
            train_auto(m, tr, dv, out, input_noise_std=std)
    for seed in BAD_SEED:
        with pytest.raises(ValueError, match=r"noise_seed must be an int in \[0, 2\^64\)"):
            train_auto(m, tr, dv, out, input_noise_std=0.1, noise_seed=seed)
    for k, g in ((1, 0), (1, 2), (1, -1), (3, 0), (3, 4), (3, -1), (3, 1.0), (3, True), (3, "1"), (2, 3)):
        with pytest.raises(ValueError, match=rf"rollout_grad_steps must be an int in 1\.\.rollout_steps={k}"):
            train_auto(m, tr, dv, out, rollout_steps=k, rollout_grad_steps=g)
    # valid set-ups get as far as the CPU model's refusal
    for kw in (dict(rollout_steps=1, rollout_grad_steps=1, input_noise_std=0.0), dict(rollout_steps=3, rollout_grad_steps=1),
               dict(rollout_steps=3, rollout_grad_steps=3, input_noise_std=0.5, noise_seed=2 ** 64 - 1),
               dict(input_noise_std=np.float32(0.25), noise_seed=np.uint64(7))):
        with pytest.raises(_lib.FnoNativeError, match="CPU"):
            train_auto(m, tr, dv, out, **kw)
    assert not out.exists()   # rejected before anything was written
    assert "train_auto" in cfdbench_b200.__all__
