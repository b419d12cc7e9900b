"""INTEGRATION.md section B, executed: the UNMODIFIED reference hook.c + client.c with the binding that section
shows (oracle/bind_reference.py applies it in a temporary directory and leaves only oracle/_ref/libnvshare_bound.so)
linked against our C-ABI library libnvs_engine.so.  Two oversubscribed clients under the REFERENCE daemon: the
reference's interposer, gate, protocol and threads, our data path -- allocations come from the engine (VMM chunks,
not managed memory), every hand-off evicts and fetches through nvs_evict / nvs_fetch_all, and every word comes
back (an access to an evicted slab is a SIGSEGV on the fake driver)."""
from __future__ import annotations

import json
import re
import subprocess
import sys

import pytest

from nvs_testlib import ORACLE, ROOT, Daemon, fake_env, with_ref_shim

pytestmark = pytest.mark.reference
BOUND = ORACLE / "libnvshare_bound.so"


@pytest.fixture(scope="module")
def bound(artefacts):
    r = subprocess.run([sys.executable, str(ROOT / "oracle" / "bind_reference.py")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    if not BOUND.exists():
        pytest.skip("reference sources not present and no prebuilt bound library")
    return BOUND


def test_the_bound_library_is_the_references_plus_our_c_abi(bound):
    dyn = subprocess.run(["readelf", "-d", str(bound)], capture_output=True, text=True).stdout
    assert "libnvs_engine.so" in dyn and "Library soname: [libnvshare.so]" in dyn
    syms = subprocess.run(["nm", "-D", "--undefined-only", str(bound)], capture_output=True, text=True).stdout
    used = set(re.findall(r"\bnvs_\w+", syms))
    # the whole binding: six calls of include/nvshare_engine.h (+ the config default)
    assert used == {"nvs_engine_default_config", "nvs_engine_create", "nvs_alloc", "nvs_free", "nvs_fetch_all", "nvs_evict",
                    "nvs_set_resident_mode"}, used


def test_two_oversubscribed_clients_under_the_reference_daemon(bound, default_sock_lock, tmp_path):
    d = Daemon("reference", default_sock_lock, log_path=tmp_path / "sched.log")
    try:
        procs = []
        d.ctl("-T", "1")
        for i in (1, 2):
            env = fake_env(total_mib=200, ledger=tmp_path / "hbm", trace=tmp_path / f"trace{i}.txt",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32, "NVSHARE_DEBUG": 1,
                                  "NVSHARE_STATS_FILE": tmp_path / f"stats{i}.jsonl"})
            env["LD_PRELOAD"] = with_ref_shim(bound)
            procs.append(subprocess.Popen([str(ORACLE / "driver_app"), "40", "4.0", str(i), "3"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=120) for p in procs]
    finally:
        for p in procs:                     # (a client that is still there after a failure must not outlive the test)
            if p.poll() is None:
                p.kill()
        d.stop()
    for i, (p, (out, err)) in enumerate(zip(procs, outs), 1):
        assert p.returncode == 0 and re.search(r"RESULT PASS iters=\d+ mismatches=0", out), out + err[-2500:]
        trace = (tmp_path / f"trace{i}.txt").read_text()
        assert "cuMemAllocManaged" not in trace and "cuMemCreate" in trace        # the engine's memory, not UVM
        ops = [json.loads(l)["op"] for l in (tmp_path / f"stats{i}.jsonl").read_text().splitlines()]
        assert ops.count("evict") >= 1 and ops.count("fetch") >= 2                # hand-offs went through the C-ABI
        assert "[NVSHARE][DEBUG]: Received LOCK_OK" in err                        # the reference's own client code ran


@pytest.fixture(scope="module")
def bound_opt(artefacts):
    out = ORACLE / "libnvshare_bound_opt.so"
    r = subprocess.run([sys.executable, str(ROOT / "oracle" / "bind_reference.py"), "--optional"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    if not out.exists():
        pytest.skip("reference sources not present and no prebuilt bound library")
    return out


def test_optional_calls_a_loading_client_needs_no_lock(bound_opt, default_sock_lock, tmp_path):
    """The optional one-liners of INTEGRATION.md B in the reference's own hook: with `nvs_host_io` in front of the gate
    of cuMemcpyHtoD / DtoH a client that only uploads and reads back never asks the REFERENCE daemon for the lock
    while another client holds it for a 30 s quantum (the unbound reference would wait for that quantum, src/hook.c:843)."""
    import time
    syms = subprocess.run(["nm", "-D", "--undefined-only", str(bound_opt)], capture_output=True, text=True).stdout
    assert {"nvs_host_io", "nvs_touch", "nvs_evict_announce", "nvs_gpu_lent_bytes"} <= set(re.findall(r"\bnvs_\w+", syms))
    d = Daemon("reference", default_sock_lock, log_path=tmp_path / "sched.log")
    a = None
    try:
        d.ctl("-T", "30")

        def env_for():
            env = fake_env(total_mib=200, ledger=tmp_path / "hbm",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32, "NVSHARE_DEBUG": 1})
            env["LD_PRELOAD"] = with_ref_shim(bound_opt)
            return env
        a = subprocess.Popen([str(ORACLE / "driver_app"), "40", "4.0", "1", "3"], env=env_for(),
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        time.sleep(1.0)                                   # A holds the lock and 120 of the 200 MiB by now
        t0 = time.time()
        b = subprocess.run([str(ORACLE / "load_app"), "40", "3", "9"], env=env_for(), capture_output=True, text=True, timeout=60)
        took = time.time() - t0
        out_a, err_a = a.communicate(timeout=60)
        assert a.returncode == 0 and "RESULT PASS" in out_a, out_a + err_a[-1500:]
    finally:
        if a is not None and a.poll() is None:
            a.kill()
        d.stop()
    assert b.returncode == 0 and re.search(r"RESULT PASS seconds=\S+ mismatches=0", b.stdout), b.stdout + b.stderr[-1500:]
    assert took < 2.5                                     # A still had > 2.5 s of compute and a 30 s quantum left
    assert d.read_log().count("Received REQ_LOCK") == 1   # A's; the loader never asked
