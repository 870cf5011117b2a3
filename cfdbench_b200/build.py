"""Build libcfdbench_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m cfdbench_b200.build [--force] [--verbose]

The .so and the object files are git-ignored build products.  The product path never
JIT-compiles and never falls back: if the library is missing, `cfdbench_b200._lib` raises.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libcfdbench_b200.so")
STAMP = os.path.join(HERE, ".build_stamp")
SOURCES = ["fno_abi.cu", "fno_dft_fwd.cu", "fno_dft_fwd_tc.cu", "fno_mode_mix.cu", "fno_block_tc.cu", "fno_block_fused.cu", "fno_pointwise.cu", "fno_project_tc.cu", "fno_project_bwd_tc.cu",
           "fno_backward.cu", "fno_metrics.cu", "fno_train_step.cu", "fno_grid.cu"]
NVCC_FLAGS = ["-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
              "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return "nvcc"


def _fingerprint() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def ensure_codelets() -> None:
    hdr = os.path.join(CSRC, "fft_codelets.cuh")
    gen = os.path.join(CSRC, "gen_codelets.py")
    if not os.path.exists(hdr) or os.path.getmtime(hdr) < os.path.getmtime(gen):
        subprocess.check_call([sys.executable, gen, "-o", hdr])


def build(force: bool = False, verbose: bool = False) -> str:
    ensure_codelets()
    fp = _fingerprint()
    if not force and os.path.exists(OUT) and os.path.exists(STAMP) and open(STAMP).read().strip() == fp:
        return OUT
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    objs, procs = [], []
    t0 = time.time()
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in srcs:
        o = os.path.join(HERE, "build", os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", s, "-o", o] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed for {s}\n{out}\n")
        elif verbose:
            print(f"--- {os.path.basename(s)}\n{out}")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    subprocess.check_call([_nvcc(), "-shared", "-o", OUT, *objs, "-lcudart"])
    with open(STAMP, "w") as f:
        f.write(fp)
    if verbose:
        print(f"built {OUT} in {time.time() - t0:.1f}s")
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or "-v" in sys.argv)
    print(OUT)
