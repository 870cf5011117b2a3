"""TEST INFRASTRUCTURE -- place the unmodified reference tree (luo-yining/CFDBench `src/`) in the git-ignored
oracle/_ref/src, where `bench.py --impl reference`, bench.py's `cpu_baseline`, oracle/make_golden.py and
tests/test_gpu_runner.py import it from.

The reference is a script tree without setup.py / pyproject.toml, so there is nothing to compile or pip-install: the
recipe is a copy.  The checkout is the one the CFDBENCH_REFERENCE environment variable names, else the default location
DEFAULT_REF when it exists there; with neither nothing is installed, tests/test_gpu_runner.py skips and bench.py times
the verified torch port instead.  Nothing under oracle/_ref is committed or read by the product path.

    [CFDBENCH_REFERENCE=/path/to/CFDBench] python oracle/install_reference.py
"""
from __future__ import annotations

import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref", "src")
DEFAULT_REF = "/root/reference"   # where the build environment keeps its CFDBench checkout


def install() -> str | None:
    ref = os.environ.get("CFDBENCH_REFERENCE")
    if ref:
        src = os.path.join(ref, "src")
        if not os.path.isdir(os.path.join(src, "models", "fno")):
            raise FileNotFoundError(f"CFDBENCH_REFERENCE={ref}: no src/models/fno in it")
    else:
        src = os.path.join(DEFAULT_REF, "src")
        if not os.path.isdir(os.path.join(src, "models", "fno")):
            return None
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    shutil.copytree(src, DST, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    return DST


if __name__ == "__main__":
    print(install() or f"no reference checkout (CFDBENCH_REFERENCE unset, nothing at {DEFAULT_REF}): nothing installed")
