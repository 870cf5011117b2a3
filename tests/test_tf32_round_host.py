"""tc::round_tf32 and tc::split_tf32 (cfdbench_b200/csrc/tf32_round.cuh), compiled for the host from the shipped header
and checked on all 2^32 fp32 bit patterns:

  * not NaN: the bits of the bit trick (u + 0x1000) & 0xffffe000 -- so every finite kernel output and every constant
    table built from it is unchanged by the NaN handling;
  * finite: also an independent definition, computed in double: round half away from zero to the tf32 grid, spacing
    max(2^(e - 11), 2^-136) for |x| in [2^(e-1), 2^e) (frexp's e), +-Inf from 2^128 on, the sign kept (also on +-0);
  * NaN: a NaN with its 13 low bits zero (the tensor core truncates those when it reads an operand, so a NaN with its
    payload only there would be read as Inf);
  * split_tf32, finite x below the overflow threshold 0x7f7ff000: hi and lo are tf32 values and
    |x - hi - lo| <= 2^-22 |x| + 2^-137 (half of tf32's subnormal spacing); NaN x: hi is NaN.

The same sweep run on the bare bit trick must find NaN failures and nothing else, which shows the NaN checks can fail.
`-s` prints the sweep's time."""
import ctypes
import os
import subprocess
import tempfile
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHIM = r'''
#include <math.h>
#include <stdint.h>
#include <thread>
#include <vector>
#include "tf32_round.cuh"

static inline float bare_round(float x) {   // the bit trick without the NaN test
  return fno::tc::f32_from_bits((fno::tc::f32_bits(x) + 0x1000u) & 0xffffe000u);
}
static inline void bare_split(float x, float& hi, float& lo) { hi = bare_round(x); lo = bare_round(x - hi); }

enum { kNonNanBits, kFiniteIndependent, kNanResult, kSplitTf32, kSplitBound, kSplitNan, kChecks };

// the tf32 grid spacing of x: max(2^(e - 11), 2^-136), |x| in [2^(e-1), 2^e)
static double tf32_spacing(float x) {
  int e;
  frexp(static_cast<double>(x), &e);
  return ldexp(1.0, e - 11 > -136 ? e - 11 : -136);
}
// round half away from zero to the grid of spacing s, in double
static float independent_round(float x, double s) {
  if (x == 0.0f) return x;
  const double r = floor(fabs(static_cast<double>(x)) / s + 0.5) * s;
  const float m = r >= ldexp(1.0, 128) ? INFINITY : static_cast<float>(r);
  return copysignf(m, x);
}

template <bool kBare>
static void sweep_range(uint64_t lo_u, uint64_t hi_u, uint64_t* count, uint32_t* first) {
  uint32_t binade = ~0u;   // the exponent field the spacing below was computed for (one spacing per field, 0 included)
  double s = 0.0;
  for (uint64_t v = lo_u; v < hi_u; ++v) {
    const uint32_t u = static_cast<uint32_t>(v);
    const float x = fno::tc::f32_from_bits(u);
    if ((u & 0x7f800000u) != binade) {
      binade = u & 0x7f800000u;
      s = tf32_spacing(fno::tc::f32_from_bits(u | 0x00400000u));   // a nonzero member of the binade
    }
    const float r = kBare ? bare_round(x) : fno::tc::round_tf32(x);
    const uint32_t rb = fno::tc::f32_bits(r);
    const bool nan = (u & 0x7fffffffu) > 0x7f800000u;
    bool bad[kChecks] = {};
    if (!nan) {
      bad[kNonNanBits] = rb != ((u + 0x1000u) & 0xffffe000u);
      if ((u & 0x7f800000u) != 0x7f800000u) bad[kFiniteIndependent] = rb != fno::tc::f32_bits(independent_round(x, s));
    } else {
      bad[kNanResult] = r == r || (rb & 0x1fffu) != 0;
    }
    float hi, lo;
    if (kBare) bare_split(x, hi, lo); else fno::tc::split_tf32(x, hi, lo);
    if (nan) {
      bad[kSplitNan] = hi == hi;
    } else if ((u & 0x7fffffffu) < 0x7f7ff000u) {
      bad[kSplitTf32] = ((fno::tc::f32_bits(hi) | fno::tc::f32_bits(lo)) & 0x1fffu) != 0;
      const double xd = x, err = fabs(xd - static_cast<double>(hi) - static_cast<double>(lo));
      bad[kSplitBound] = !(err <= ldexp(fabs(xd), -22) + ldexp(1.0, -137));
    }
    for (int k = 0; k < kChecks; ++k)
      if (bad[k] && count[k]++ == 0) first[k] = u;
  }
}

extern "C" int tf32_checks() { return kChecks; }

// counts[k] = failures of check k, first[k] = the first failing pattern; bare != 0 sweeps the bit trick alone
extern "C" void tf32_sweep(int bare, int n_threads, uint64_t* counts, uint32_t* first) {
  std::vector<std::vector<uint64_t>> c(n_threads, std::vector<uint64_t>(kChecks, 0));
  std::vector<std::vector<uint32_t>> f(n_threads, std::vector<uint32_t>(kChecks, 0));
  std::vector<std::thread> pool;
  const uint64_t n = 1ull << 32, per = (n + n_threads - 1) / n_threads;
  for (int t = 0; t < n_threads; ++t) {
    const uint64_t a = per * t, b = per * (t + 1) < n ? per * (t + 1) : n;
    pool.emplace_back([=, &c, &f] {
      if (bare) sweep_range<true>(a, b, c[t].data(), f[t].data());
      else sweep_range<false>(a, b, c[t].data(), f[t].data());
    });
  }
  for (auto& th : pool) th.join();
  for (int k = 0; k < kChecks; ++k) {
    counts[k] = 0;
    for (int t = n_threads - 1; t >= 0; --t)
      if (c[t][k]) { counts[k] += c[t][k]; first[k] = f[t][k]; }
  }
}
'''

CHECKS = ["non-NaN: bits of (u + 0x1000) & 0xffffe000", "finite: the independent float64 rounding",
          "NaN: a NaN with 13 zero low bits", "split: hi and lo are tf32", "split: |x - hi - lo| bound",
          "split: NaN hi"]
NAN_CHECKS = {2, 5}


@pytest.fixture(scope="module")
def tf32_lib():
    d = tempfile.mkdtemp(prefix="fno_tf32_")
    src, so = os.path.join(d, "tf32.cpp"), os.path.join(d, "tf32.so")
    with open(src, "w") as f:
        f.write(SHIM)
    # no -ffast-math: the NaN test in round_tf32 and the reference's NaN checks need IEEE compares
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-ffp-contract=off",
                           "-I", os.path.join(ROOT, "cfdbench_b200", "csrc"), src, "-o", so])
    lib = ctypes.CDLL(so)
    assert lib.tf32_checks() == len(CHECKS)
    return lib


def _sweep(lib, bare):
    counts, first = (ctypes.c_uint64 * len(CHECKS))(), (ctypes.c_uint32 * len(CHECKS))()
    t0 = time.time()
    lib.tf32_sweep(int(bare), max(1, min(os.cpu_count() or 1, 16)), counts, first)
    dt = time.time() - t0
    fails = {CHECKS[k]: (counts[k], f"0x{first[k]:08x}") for k in range(len(CHECKS)) if counts[k]}
    return fails, {k for k in range(len(CHECKS)) if counts[k]}, dt


def test_round_tf32_on_every_bit_pattern(tf32_lib):
    fails, _, dt = _sweep(tf32_lib, bare=False)
    print(f"\n[tf32 sweep] 2^32 patterns in {dt:.1f} s")
    assert not fails, f"(failures, first failing pattern) per check: {fails}"


def test_the_nan_checks_catch_the_bare_bit_trick(tf32_lib):
    """The bare (u + 0x1000) & 0xffffe000 passes every check but the NaN ones, which it fails: 0x7fffffff -> -0.0,
    0xffffffff -> +0.0, 0x7f800001 -> +Inf."""
    fails, failed, dt = _sweep(tf32_lib, bare=True)
    print(f"\n[tf32 sweep, bare bit trick] {dt:.1f} s: {fails}")
    assert failed == NAN_CHECKS, fails
