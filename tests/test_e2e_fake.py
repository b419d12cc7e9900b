"""Whole stack on CPU: nvshare-scheduler + N unmodified driver-API applications
(tests/apps/driver_app.c) with libnvshare.so injected by LD_PRELOAD, against
oracle/fake_cuda.c with a SHARED physical-memory ledger so that the clients are
genuinely oversubscribed: client B cannot map its working set until client A
has released HBM, and an access to an evicted slab is a SIGSEGV.

Also the interoperability matrix: our library under the reference daemon and
the reference library under our daemon (wire compatibility both ways).
"""
from __future__ import annotations

import re
import subprocess

import pytest

from nvs_testlib import ORACLE, Daemon, fake_env, preload


def run_clients(daemon_impl, lib_impl, sock_dir, tmp_path, n_clients=2, mib=40, nbuf=3, seconds=4.0, total_mib=200,
                tq=1, extra=None):
    d = Daemon(daemon_impl, sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", str(tq))
        procs = []
        for i in range(n_clients):
            env = fake_env(total_mib=total_mib, ledger=tmp_path / "ledger",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32,
                                  "NVSHARE_DEBUG": 1, **(extra or {})})
            env["LD_PRELOAD"] = preload(lib_impl)
            if daemon_impl == "ours":
                env["NVSHARE_SOCK_DIR"] = str(sock_dir)
            procs.append(subprocess.Popen([str(ORACLE / "driver_app"), str(mib), str(seconds), str(i + 1), str(nbuf)],
                                          env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=120) for p in procs]
        return d.read_log(), [(p.returncode, o, e) for p, (o, e) in zip(procs, outs)]
    finally:
        d.stop()


def check(results):
    for rc, out, err in results:
        assert rc == 0, out + err[-2000:]
        assert re.search(r"RESULT PASS iters=\d+ mismatches=0", out), out


def test_two_clients_oversubscribed(artefacts, sock_dir, tmp_path):
    # 2 x 120 MiB of allocations on a 200 MiB "GPU": 1.2x oversubscribed
    log, results = run_clients("ours", "ours", sock_dir, tmp_path)
    check(results)
    assert log.count("Sent DROP_LOCK") >= 3
    evicts = [len(re.findall(r"engine: evict", err)) for _, _, err in results]
    fetches = [len(re.findall(r"engine: fetch", err)) for _, _, err in results]
    assert min(evicts) >= 1 and min(fetches) >= 2           # both clients were swapped out and came back


def test_three_clients_late_release_order(artefacts, sock_dir, tmp_path):
    # eviction completes BEFORE LOCK_RELEASED (no overlap): the conservative ordering must work too
    log, results = run_clients("ours", "ours", sock_dir, tmp_path, n_clients=3, mib=30, seconds=5.0,
                               extra={"NVSHARE_EARLY_RELEASE": 0})
    check(results)


@pytest.mark.parametrize("variant", ["ldg", "ce"])
def test_other_copy_variants(artefacts, sock_dir, tmp_path, variant):
    log, results = run_clients("ours", "ours", sock_dir, tmp_path, seconds=3.0,
                               extra={"NVSHARE_COPY_VARIANT": variant})
    check(results)


def test_uvm_mode_two_clients(artefacts, sock_dir, tmp_path):
    # the reference's mechanism, kept as a mode: managed memory never touches the ledger
    log, results = run_clients("ours", "ours", sock_dir, tmp_path, seconds=3.0, extra={"NVSHARE_ENGINE": "uvm"})
    check(results)
    assert all("engine:" not in err for _, _, err in results)


def test_gpu_without_our_kernel_image_runs_on_managed_memory(artefacts, sock_dir, tmp_path):
    """ADVICE r1: only the sm_90a image is embedded; on any other GPU the drop-in must still work.  The engine
    fails to load its kernels, the library says so and runs the process on the reference's mechanism."""
    log, results = run_clients("ours", "ours", sock_dir, tmp_path, seconds=3.0, extra={"FAKE_CUDA_NO_BINARY": 1})
    check(results)
    for _, _, err in results:
        assert "swap engine unavailable on this GPU/driver" in err and "managed-memory mechanism" in err


@pytest.mark.reference
def test_our_library_under_reference_daemon(artefacts, default_sock_lock, tmp_path):
    log, results = run_clients("reference", "ours", default_sock_lock, tmp_path, seconds=3.0)
    check(results)
    assert log.count("Sent DROP_LOCK") >= 2


@pytest.mark.reference
def test_reference_library_under_our_daemon(artefacts, default_sock_lock, tmp_path):
    # the reference library only knows /var/run/nvshare: run OUR daemon there
    import os
    d = None
    old = os.environ.get("NVSHARE_SOCK_DIR")
    os.environ["NVSHARE_SOCK_DIR"] = str(default_sock_lock)
    try:
        log, results = run_clients("ours", "reference", default_sock_lock, tmp_path, seconds=3.0)
    finally:
        if old is None:
            os.environ.pop("NVSHARE_SOCK_DIR", None)
        else:
            os.environ["NVSHARE_SOCK_DIR"] = old
    check(results)
    assert log.count("Sent DROP_LOCK") >= 2


def test_anti_thrash_off_and_on_again(artefacts, sock_dir, tmp_path):
    """nvsharectl -S off lets every client run at once (they must all fit: 2 x 120 MiB on
    400 MiB); -S on closes the gates again.  Data survive both transitions."""
    import time
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "1")
        procs = []
        for i in (1, 2):
            env = fake_env(total_mib=400, ledger=tmp_path / "ledger",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_DEBUG": 1,
                                  "NVSHARE_SOCK_DIR": sock_dir, "NVSHARE_POOL_GIB": 1})
            env["LD_PRELOAD"] = preload("ours")
            procs.append(subprocess.Popen([str(ORACLE / "driver_app"), "40", "6", str(i), "3"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        time.sleep(2.0)
        d.ctl("-S", "off")
        time.sleep(2.0)
        d.ctl("-S", "on")
        outs = [p.communicate(timeout=120) for p in procs]
    finally:
        d.stop()
    for p, (out, err) in zip(procs, outs):
        assert p.returncode == 0 and re.search(r"RESULT PASS iters=\d+ mismatches=0", out), out + err[-2500:]
        assert "Scheduler status changed to OFF" in err and "Scheduler status changed to ON" in err


@pytest.mark.parametrize("io", [0, 1])
def test_multithreaded_clients_oversubscribed(artefacts, sock_dir, tmp_path, io):
    """Four application threads per client issue copies and launches concurrently while
    the lock changes hands every second: nothing may touch a slab that is being unmapped
    (the fake driver would segfault) and every thread's data must survive.  io=1: each
    thread also reads back, checks and rewrites a buffer every iteration -- copies that are
    served by the device path or from the backing copy (nvs_host_io) depending on where the
    lock happens to be, and must agree with each other."""
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "1")
        procs = []
        for i in (1, 2):
            env = fake_env(total_mib=200, ledger=tmp_path / "ledger",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32,
                                  "NVSHARE_DEBUG": 1, "NVSHARE_SOCK_DIR": sock_dir, "NVSHARE_POOL_GIB": 1})
            env["LD_PRELOAD"] = preload("ours")
            # 4 threads x 2 buffers x 16 MiB = 128 MiB per client on a 200 MiB "GPU"
            procs.append(subprocess.Popen([str(ORACLE / "mt_app"), "16", "5", str(i), "4", str(io)], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=120) for p in procs]
    finally:
        d.stop()
    for p, (out, err) in zip(procs, outs):
        assert p.returncode == 0 and re.search(r"RESULT PASS iters=\d+ mismatches=0", out), out + err[-2500:]
    assert d.read_log().count("Sent DROP_LOCK") >= 3
    if io:
        served = sum(err.count("served from the backing copy") for _, err in outs)
        assert served >= 1                                   # both paths were really taken
        assert sum(err.count("Sent REQ_LOCK") for _, err in outs) >= 4


def test_client_exits_when_scheduler_is_absent(artefacts, sock_dir, tmp_path):
    env = fake_env(extra={"NVSHARE_SOCK_DIR": sock_dir})
    env["LD_PRELOAD"] = preload("ours")
    r = subprocess.run([str(ORACLE / "driver_app"), "4", "0.1", "1"], env=env, capture_output=True, text=True,
                       timeout=30)
    assert r.returncode == 1                                 # reference: exit(1) in the host app (client.c:250)
    assert "[NVSHARE][FATAL]" in r.stderr


def _loader_beside_a_holder(sock_dir, tmp_path, lockfree):
    """Client A computes and holds the lock for a long quantum; client B only
    allocates, uploads and reads back (tests/apps/load_app.c)."""
    import time
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "30")
        def env_for():
            env = fake_env(total_mib=200, ledger=tmp_path / "ledger",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32,
                                  "NVSHARE_DEBUG": 1, "NVSHARE_LOCKFREE_COPY": int(lockfree)})
            env["LD_PRELOAD"] = preload("ours")
            env["NVSHARE_SOCK_DIR"] = str(sock_dir)
            return env
        a = subprocess.Popen([str(ORACLE / "driver_app"), "40", "4.0", "1", "3"], env=env_for(),
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        time.sleep(1.0)                                   # A holds the lock and 120 of the 200 MiB by now
        t0 = time.time()
        b = subprocess.run([str(ORACLE / "load_app"), "40", "3", "9"], env=env_for(), capture_output=True, text=True,
                           timeout=60)
        took = time.time() - t0
        out_a, err_a = a.communicate(timeout=60)
        assert a.returncode == 0 and "RESULT PASS" in out_a, out_a + err_a[-1500:]
        return b, took
    finally:
        d.stop()


def test_loading_client_does_not_need_the_lock(artefacts, sock_dir, tmp_path):
    """SURVEY 8f rank 3: uploads to (and reads from) memory that is not on the GPU
    are served from the pinned-host backing copy; the loading client never asks
    for the lock, so it neither waits for the holder nor takes the GPU from it."""
    b, took = _loader_beside_a_holder(sock_dir, tmp_path, lockfree=True)
    assert b.returncode == 0 and re.search(r"RESULT PASS seconds=\S+ mismatches=0", b.stdout), b.stdout + b.stderr[-1500:]
    assert "Sent REQ_LOCK" not in b.stderr                 # not once
    assert b.stderr.count("served from the backing copy") >= 12
    assert took < 2.5                                      # A still had >2.5 s of compute and a 30 s quantum left


def test_loading_client_waits_when_the_bypass_is_off(artefacts, sock_dir, tmp_path):
    """The reference's behaviour (src/hook.c:843-971), kept behind NVSHARE_LOCKFREE_COPY=0:
    the first copy waits for the lock, i.e. until A goes idle and releases it."""
    b, took = _loader_beside_a_holder(sock_dir, tmp_path, lockfree=False)
    assert b.returncode == 0 and "RESULT PASS" in b.stdout, b.stdout + b.stderr[-1500:]
    assert "Sent REQ_LOCK" in b.stderr and "served from the backing copy" not in b.stderr
    assert took > 2.5


@pytest.mark.parametrize("policy", ["all", "need"])
def test_tight_backing_pool_makes_progress(artefacts, sock_dir, tmp_path, policy):
    """The shared pool (128 MiB) is smaller than what the two clients put into it when
    both are swapped out (2 x 120 MiB with the evict-all policy): the releasing client's
    eviction has to wait for units that only the next holder's fetch returns -- hand-offs
    must keep flowing (regression: two clients evicting at once once filled the pool and
    waited for each other until the time-out, profiles/r01_call19_deadlock_diagnostics.json)."""
    log, results = run_clients("ours", "ours", sock_dir, tmp_path, seconds=6.0,
                               extra={"NVSHARE_POOL_MIB": 128, "NVSHARE_EVICT_POLICY": policy,
                                      "NVSHARE_OOM_WAIT_MS": 8000})
    check(results)
    assert log.count("Sent DROP_LOCK") >= 4
    for _, _, err in results:
        assert "backing tier exhausted" not in err and "timed out" not in err


def test_pool_too_small_for_three_clients_overflows_instead_of_failing(artefacts, sock_dir, tmp_path):
    """Three multi-threaded clients of ~84 MiB on a 200 MiB "GPU" with the evict-all policy
    keep two of them fully swapped out (168 MiB) -- more than the 128 MiB shared pool can
    ever hold.  After a grace period the evicting client pins a private overflow arena
    beside the pool; every hand-off completes and every byte survives."""
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "1")
        procs = []
        for i in (1, 2, 3):
            env = fake_env(total_mib=200, ledger=tmp_path / "ledger",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32,
                                  "NVSHARE_DEBUG": 1, "NVSHARE_SOCK_DIR": sock_dir, "NVSHARE_POOL_MIB": 128,
                                  "NVSHARE_EVICT_POLICY": "all", "NVSHARE_OOM_WAIT_MS": 15000})
            env["LD_PRELOAD"] = preload("ours")
            procs.append(subprocess.Popen([str(ORACLE / "mt_app"), "12", "8", str(i), "3", "1"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=180) for p in procs]
    finally:
        d.stop()
    for p, (out, err) in zip(procs, outs):
        assert p.returncode == 0 and re.search(r"RESULT PASS iters=\d+ mismatches=0", out), out + err[-2500:]
    # whether the overflow arena is really needed depends on timing (units may come back within the grace
    # period; kept copies are taken over first): tests/test_engine_fake.py pins that path deterministically.
    # Here: nobody failed, nobody timed out.
    for _, err in outs:
        assert "backing tier exhausted" not in err and "timed out" not in err
    assert d.read_log().count("Sent DROP_LOCK") >= 4


def test_stream_ordered_and_pitched_allocations_are_capped_and_swapped(artefacts, sock_dir, tmp_path):
    """SURVEY 8f rank 2 / VERDICT r1 #8: cuMemAllocAsync, cuMemAllocFromPoolAsync, cuMemFreeAsync and
    cuMemAllocPitch go through the cap check and the swap engine like cuMemAlloc (the reference lets
    them through: such memory is neither charged nor swappable there)."""
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "1")
        procs = []
        for i in (1, 2):
            env = fake_env(total_mib=4096, ledger=tmp_path / "ledger", trace=tmp_path / f"trace{i}.txt",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_SOCK_DIR": sock_dir,
                                  "NVSHARE_POOL_GIB": 1, "NVSHARE_EVICT_POLICY": "all",
                                  "NVSHARE_STATS_FILE": tmp_path / f"stats{i}.jsonl"})
            env["LD_PRELOAD"] = preload("ours")
            procs.append(subprocess.Popen([str(ORACLE / "async_app"), "16", "3.0", str(i), "3"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=120) for p in procs]
    finally:
        d.stop()
    import json
    for i, (p, (out, err)) in enumerate(zip(procs, outs), 1):
        assert p.returncode == 0 and "RESULT PASS" in out, out + err[-2000:]
        assert "CAP rc=2" in out                       # 3 GiB > 4096 - 1536 MiB: CUDA_ERROR_OUT_OF_MEMORY, like cuMemAlloc
        assert "WRAP rc=2" in out                      # sum + request wraps around 2^64: still refused
        trace = (tmp_path / f"trace{i}.txt").read_text()
        assert "cuMemAllocAsync" not in trace and "cuMemAllocPitch" not in trace and "cuMemCreate" in trace
        ops = [json.loads(l)["op"] for l in (tmp_path / f"stats{i}.jsonl").read_text().splitlines()]
        assert "evict" in ops and "fetch" in ops       # and it is swapped like any other memory


def _capture_run(impl, sd, tmp_path):
    d = Daemon(impl, sd)
    try:
        env = fake_env(total_mib=4096, trace=tmp_path / f"trace_{impl}.txt",
                       extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_SOCK_DIR": sd})
        env["LD_PRELOAD"] = preload(impl)
        r = subprocess.run([str(ORACLE / "capture_app"), "5000"], env=env, capture_output=True, text=True, timeout=120)
        return r.returncode, r.stdout, r.stderr, (tmp_path / f"trace_{impl}.txt").read_text()
    finally:
        d.stop()


def test_stream_capture_survives_the_sync_window(artefacts, sock_dir, tmp_path):
    """SURVEY 8f rank 2 / DESIGN 8: a launch into a capturing stream records a graph node; synchronising then is an
    illegal call that invalidates the capture.  5000 captured launches (more than any sync window) leave the capture
    intact, and a stream-ordered free of swappable memory inside it is refused (801) without harming it."""
    rc, out, err, trace = _capture_run("ours", sock_dir, tmp_path)
    assert rc == 0 and "RESULT PASS" in out, out + err[-2000:]
    assert "FREE_IN_CAPTURE rc=801" in out and "END_CAPTURE rc=0" in out and "FREE_AFTER rc=0" in out
    assert "during capture" not in trace


@pytest.mark.reference
def test_stream_capture_breaks_under_the_reference_library(artefacts, default_sock_lock, tmp_path):
    """The documented difference: the reference synchronises every `window` launches regardless of capture
    (src/hook.c:808), which invalidates the capture of the same application."""
    rc, out, err, trace = _capture_run("reference", default_sock_lock, tmp_path)
    # its cuLaunchKernel hook hands the failed synchronisation back to the application (or, had the application
    # ignored that, the capture would have ended as invalidated)
    assert rc != 0 and ("cuLaunchKernel" in out and "-> 900" in out or "END_CAPTURE rc=901" in out), out + err[-2000:]
    assert "cuCtxSynchronize during capture" in trace


def test_allocation_from_a_second_context_is_not_served_by_the_first_contexts_engine(artefacts, sock_dir, tmp_path):
    """The reference assumes one context and one device, but its managed memory does not care which context asks
    for it; an engine of ours lives in ONE context on ONE GPU.  A process that creates a second context (a second
    GPU) gets managed memory there, like under the reference, loudly -- never memory of the wrong GPU."""
    d = Daemon("ours", sock_dir)
    try:
        env = fake_env(total_mib=4096, devices=2, trace=tmp_path / "trace.txt",
                       extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_SOCK_DIR": sock_dir,
                              "NVSHARE_POOL": "private"})
        env["LD_PRELOAD"] = preload("ours")
        r = subprocess.run([str(ORACLE / "two_ctx_app")], env=env, capture_output=True, text=True, timeout=60)
    finally:
        d.stop()
    assert r.returncode == 0 and "RESULT PASS" in r.stdout, r.stdout + r.stderr[-2000:]
    assert r.stderr.count("allocation from a second CUDA context") == 1
    trace = (tmp_path / "trace.txt").read_text()
    assert trace.count("cuMemAllocManaged 4194304") == 1          # the second context's buffer, and only that one
    assert trace.count("cuMemCreate") >= 2                        # the first context's two buffers: engine memory


@pytest.mark.parametrize("peers", ["1", "auto"])
def test_hooked_clients_on_the_peer_tier(artefacts, sock_dir, tmp_path, peers):
    """The peer-HBM backing tier through the interposer (NVSHARE_PEERS in the application's environment, the way
    bench.py --gpus N sets it): two oversubscribed clients of "GPU 0" back their slabs on "GPU 1" of the fake driver
    (a list of ordinals, or `auto` = every other GPU it can reach) and get every word back."""
    import json
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    procs = []
    try:
        d.ctl("-T", "1")
        for i in (1, 2):
            env = fake_env(total_mib=200, ledger=tmp_path / "ledger", devices=2,
                           extra={"NVSHARE_HOST_ARENA_MIB": 32, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32, "NVSHARE_DEBUG": 1,
                                  "NVSHARE_SOCK_DIR": sock_dir, "NVSHARE_PEERS": peers, "NVSHARE_GPU_LEDGER": tmp_path / "gpus",
                                  "NVSHARE_GPU_RESERVE_MIB": 8, "NVSHARE_STATS_FILE": tmp_path / f"stats{i}.jsonl"})
            env["LD_PRELOAD"] = preload("ours")
            procs.append(subprocess.Popen([str(ORACLE / "driver_app"), "40", "4.0", str(i), "3"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=120) for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        d.stop()
    check([(p.returncode, o, e) for p, (o, e) in zip(procs, outs)])
    for i in (1, 2):
        recs = [json.loads(l) for l in (tmp_path / f"stats{i}.jsonl").read_text().splitlines()]
        ev = [r for r in recs if r["op"] == "evict"]
        assert ev and sum(r["peer_bytes"] for r in ev) > 0                    # slabs went to the other GPU's HBM
        assert all(r["gl_tracked_peers"] == 1 for r in ev)                    # and the ledger knows whose it is
        assert max(r["gl_lent"] for r in ev) <= (200 - 8) << 20
    if peers == "auto":
        assert "NVSHARE_PEERS=auto: 1 peer GPU(s) of device 0" in outs[0][1]
