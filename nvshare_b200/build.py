"""Build helpers: everything is compiled in-tree by make (gcc + nvcc), no JIT.

  build_product()  nvshare_b200/csrc/Makefile -> nvshare_b200/_build/
                   {libnvshare.so, libnvs_engine.so, nvshare-scheduler, nvsharectl,
                    slab_copy.cubin}; the only CUDA TU is compiled with
                   -gencode arch=compute_90a,code=sm_90a -lineinfo
  build_oracle()   oracle/Makefile -> oracle/_ref/ (test infrastructure: the
                   unmodified reference where its sources can be read, the fake
                   driver, the C restatement, the test applications, and the
                   reference's hook + client bound to our C-ABI: libnvshare_bound.so)
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "nvshare_b200" / "csrc"
BUILD = ROOT / "nvshare_b200" / "_build"
ORACLE = ROOT / "oracle"
ORACLE_OUT = ORACLE / "_ref"

PRODUCT_ARTEFACTS = ["libnvshare.so", "libnvs_engine.so", "nvshare-scheduler", "nvsharectl", "slab_copy.cubin"]


def _run(cmd, cwd):
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"{' '.join(map(str, cmd))} failed in {cwd}:\n{r.stdout[-4000:]}")
    return r.stdout


def have_nvcc() -> bool:
    return shutil.which(os.environ.get("NVCC", "nvcc")) is not None


def build_product(force: bool = False) -> Path:
    """Compile the product.  On a box without nvcc the prebuilt artefacts that
    travelled with the tree are used as they are (and must all exist)."""
    if have_nvcc() or force:
        _run(["make", "-C", str(CSRC), "-j8"], ROOT)
    missing = [a for a in PRODUCT_ARTEFACTS if not (BUILD / a).exists()]
    if missing:
        raise RuntimeError(f"product artefacts missing and cannot be built here: {missing}")
    return BUILD


def build_oracle() -> Path:
    """Build the test infrastructure (never part of the product path)."""
    _run(["make", "-C", str(ORACLE), "all"], ROOT)
    # INTEGRATION.md section B made executable: the unmodified reference hook + client bound to our C-ABI library
    # (only where the reference's sources and our product are present; the result travels like the rest of _ref)
    if (BUILD / "libnvs_engine.so").exists():
        import sys
        _run([sys.executable, str(ORACLE / "bind_reference.py")], ROOT)
        _run([sys.executable, str(ORACLE / "bind_reference.py"), "--optional"], ROOT)
    return ORACLE_OUT


def reference_available() -> bool:
    return all((ORACLE_OUT / n).exists() for n in ("libnvshare.so", "nvshare-scheduler", "nvsharectl", "libsockdir.so"))
