"""(1) The drop-in boundary as an ELF fact: every symbol include/*.h declares is
exported by the C-ABI library, libnvshare.so exports the reference's interposed
set under the reference's symbol versions and NEEDs nothing but libc.
(2) The oracle restatement (oracle/nvshare_oracle.c) against the reference's
constants and the committed golden fixture.
No GPU, no compute calls."""
from __future__ import annotations

import ctypes as C
import json
import re
import subprocess
from pathlib import Path

import pytest

from nvs_testlib import BUILD, ORACLE, ROOT

REFERENCE_EXPORTS = [  # SURVEY 8b, probe `nm -D` on the reference's libnvshare.so
    "cuInit", "cuGetProcAddress", "cuGetProcAddress_v2", "cuMemAlloc_v2", "cuMemFree_v2", "cuMemGetInfo_v2",
    "cuLaunchKernel", "cuMemcpy", "cuMemcpyAsync", "cuMemcpyHtoD_v2", "cuMemcpyHtoDAsync_v2", "cuMemcpyDtoH_v2",
    "cuMemcpyDtoHAsync_v2", "cuMemcpyDtoD_v2", "cuMemcpyDtoDAsync_v2"]


def dynsyms(path):
    out = subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True, check=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if ln.strip()}


def test_engine_header_symbols_are_exported(artefacts):
    header = (ROOT / "include" / "nvshare_engine.h").read_text()
    declared = set(re.findall(r"^\s*(?:int|void|const char \*|uint64_t)\s*\*?\s*(nvs_\w+)\s*\(", header, re.M))
    assert {"nvs_engine_create", "nvs_alloc", "nvs_free", "nvs_evict", "nvs_fetch_all", "nvs_copy_slabs"} <= declared
    for lib in ("libnvs_engine.so", "libnvshare.so"):
        missing = declared - dynsyms(BUILD / lib)
        assert not missing, f"{lib} does not export {missing}"
    lib = C.CDLL(str(BUILD / "libnvs_engine.so"))
    for name in declared:
        getattr(lib, name)


def test_libnvshare_exports_the_reference_boundary(artefacts):
    syms = dynsyms(BUILD / "libnvshare.so")
    assert set(REFERENCE_EXPORTS) <= {s.split("@")[0] for s in syms}
    assert "dlsym@@GLIBC_2.2.5" in syms and "dlsym@GLIBC_2.34" in syms       # src/hook.c:974-975
    internals = {"continue_with_lock", "nvs_client_start", "nvs_write_all", "nvs_debug_enabled"}
    assert not (internals & {s.split("@")[0] for s in syms})


def test_exports_are_a_superset_of_the_reference_binary(artefacts):
    # driver entry points (cu + capital) and dlsym, as `nm -D` lists them for the reference's libnvshare.so
    # (tests/golden/make_golden.py); its other visible symbols (cuda_ctx, dlsym_225, ...) are accidental
    # (no `local:` in its version script)
    ref = set(json.loads((ROOT / "tests" / "golden" / "reference_exports.json").read_text()))
    ours = {s.split("@")[0] for s in dynsyms(BUILD / "libnvshare.so")}
    assert ref <= ours, ref - ours


def test_libnvshare_needs_only_libc(artefacts):
    for lib in ("libnvshare.so", "libnvs_engine.so"):
        out = subprocess.run(["readelf", "-d", str(BUILD / lib)], capture_output=True, text=True, check=True).stdout
        needed = re.findall(r"NEEDED\)\s+Shared library: \[(.+?)\]", out)
        assert needed == ["libc.so.6"], (lib, needed)        # no libcudart, no libcuda link-time dependency
    out = subprocess.run(["readelf", "-d", str(BUILD / "libnvshare.so")], capture_output=True, text=True).stdout
    assert "soname: [libnvshare.so]" in out                  # src/Makefile:19


def test_kernel_image_is_sm90a_with_bulk_copies(artefacts):
    import shutil
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not installed")
    sass = subprocess.run(["cuobjdump", "-sass", str(BUILD / "slab_copy.cubin")], capture_output=True, text=True).stdout
    assert "sm_90a" in sass or "SM90" in sass.upper()
    tma = sass.split("Function : nvs_slab_copy_tma")[1].split("Function :")[0]
    assert "UBLKCP.S.G" in tma and "UBLKCP.G.S" in tma        # cp.async.bulk both ways (TMA, non-tensor)
    assert "SYNCS.ARRIVE.TRANS64" in tma                      # mbarrier expect_tx
    ldg = sass.split("Function : nvs_slab_copy_ldg")[1].split("Function :")[0]
    assert "LDG.E.EF.128" in ldg and "STG.E.EF.128" in ldg    # 16-byte streaming vector access


# ------------------------------------------------------------------ oracle ---

@pytest.fixture(scope="module")
def orc(artefacts):
    lib = C.CDLL(str(ORACLE / "liboracle.so"))
    lib.oracle_msg_size.restype = C.c_size_t
    lib.oracle_msg_offset.restype = C.c_size_t
    lib.oracle_meminfo_free.restype = C.c_uint64
    return lib


class Book(C.Structure):
    _fields_ = [("total", C.c_uint64), ("sum_allocated", C.c_uint64), ("single_oversub", C.c_int)]


def test_oracle_wire_layout(orc):
    assert orc.oracle_msg_size() == 537                      # SURVEY section 4 probe of the reference
    assert [orc.oracle_msg_offset(i) for i in range(5)] == [0, 1, 255, 509, 517]
    import struct
    from nvs_testlib import MSG_FMT
    assert struct.calcsize(MSG_FMT) == 537


def test_oracle_bookkeeping_matches_reference_fixture(orc):
    gold = json.loads((ROOT / "tests" / "golden" / "hook_golden.json").read_text())["stdout"]
    total = 192 << 30
    b = Book(total, 0, 0)
    assert (total - orc.oracle_meminfo_free(C.byref(b))) >> 20 == 1536
    assert f"meminfo rc=0 reserve_mib=1536" in gold
    rc1 = orc.oracle_alloc(C.byref(b), C.c_uint64(100 << 30))
    rc2 = orc.oracle_alloc(C.byref(b), C.c_uint64(100 << 30))
    assert f"alloc1 rc={rc1}" in gold and f"alloc2 rc={rc2}" in gold and (rc1, rc2) == (0, 2)
    b.single_oversub = 1
    assert orc.oracle_alloc(C.byref(b), C.c_uint64(100 << 30)) == 0          # src/hook.c:663-669


def test_oracle_window_matches_reference_trace(orc):
    # fixture: launch, sync, launch, launch, sync  <=> windows 1 -> 2 -> 4 with fast syncs
    gold = json.loads((ROOT / "tests" / "golden" / "hook_golden.json").read_text())["calls"]
    pattern = [c for c in gold if c in ("cuLaunchKernel", "cuCtxSynchronize")]
    w, since, sim = 1, 0, []
    for _ in range(3):
        sim.append("cuLaunchKernel")
        since += 1
        if since >= w:
            sim.append("cuCtxSynchronize")
            w, since = orc.oracle_next_window(w, 0), 0
    assert sim == pattern and w == 4
    assert orc.oracle_next_window(2048, 0) == 2048 and orc.oracle_next_window(64, 1) == 32
    assert orc.oracle_next_window(1, 3) == 1 and orc.oracle_next_window(512, 10) == 1
