"""Test configuration.

Markers
  gpu   needs a real H100 (everything else must pass on a machine without a GPU,
        against oracle/fake_cuda.c).

Everything under oracle/ is test infrastructure: the unmodified reference built
into oracle/_ref (only where its sources are present, see oracle/Makefile), the
fake CUDA driver, the C restatement.  Product code never imports it.
"""
from __future__ import annotations

import os
import shutil
import sys
import tempfile
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from nvshare_b200 import build  # noqa: E402

# The cross-process GPU ledger (nvshare_b200/csrc/gpu_ledger.c) is one file per user and machine: the
# suite keeps its own, so that it neither sees nor leaves claims in the one real clients of this box use.
_LEDGER = Path(f"/dev/shm/nvshare-gpus-test-{os.getpid()}")
os.environ.setdefault("NVSHARE_GPU_LEDGER", str(_LEDGER))


# The daemons listen on Unix sockets under the tests' tmp_path, and a socket's path may not exceed 107 bytes:
# under a long TMPDIR or user name pytest's default base directory leaves no room for it.  The suite's temporary
# files go under a short directory of its own instead (unless --basetemp is given), removed when the run ends.
_BASETEMP = None


def pytest_sessionfinish(session, exitstatus):
    _LEDGER.unlink(missing_ok=True)
    if _BASETEMP:
        shutil.rmtree(_BASETEMP, ignore_errors=True)


def pytest_configure(config):
    global _BASETEMP
    config.addinivalue_line("markers", "gpu: needs a real H100 GPU")
    config.addinivalue_line("markers", "reference: needs the compiled reference in oracle/_ref")
    if config.option.basetemp is None:
        _BASETEMP = tempfile.mkdtemp(prefix="nvs-", dir="/tmp")
        config.option.basetemp = _BASETEMP


@pytest.fixture(scope="session")
def artefacts():
    """Build (or locate) the product and the test infrastructure once."""
    prod = build.build_product()
    try:
        orc = build.build_oracle()
    except Exception:
        orc = build.ORACLE_OUT  # GPU box without gcc headers etc.: use what travelled
    return {"build": prod, "oracle": orc, "root": ROOT}


@pytest.fixture(scope="session")
def have_reference(artefacts):
    return build.reference_available()


@pytest.fixture()
def sock_dir(tmp_path):
    d = tmp_path / "nvs"
    d.mkdir()
    return d


@pytest.fixture()
def default_sock_lock(tmp_path, monkeypatch):
    """The socket directory of a test that runs reference binaries.  They only know /var/run/nvshare, which an
    ordinary user cannot create; oracle/_ref/libsockdir.so, preloaded into them, takes NVSHARE_SOCK_DIR instead.
    It is set for the whole test, so that every client it starts -- ours or the reference's -- finds the daemon."""
    d = tmp_path / "refsock"
    d.mkdir()
    monkeypatch.setenv("NVSHARE_SOCK_DIR", str(d))
    return d


def pytest_collection_modifyitems(config, items):
    have_ref = build.reference_available()
    skip_ref = pytest.mark.skip(reason="compiled reference (oracle/_ref) not available")
    # `pytest tests` on a box without a GPU: the gpu-marked tests are skipped, not errors
    have_gpu = os.path.exists("/dev/nvidiactl") or os.path.exists("/dev/nvidia0")
    skip_gpu = pytest.mark.skip(reason="needs a real GPU (no /dev/nvidia* here)")
    for item in items:
        if item.get_closest_marker("reference") and not have_ref:
            item.add_marker(skip_ref)
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(skip_gpu)
