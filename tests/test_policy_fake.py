"""Hand-off policies that only exist between OUR library and OUR daemon (the
data-field hints of include/nvshare_wire.h), on CPU with the fake driver:
need-based partial eviction, lazy release when nobody waits, the pressure path
that makes lazy residency safe, the conservative evict-all fallback, and the
shared pinned-host pool (one backing store for all clients of a scheduler)."""
from __future__ import annotations

import os
import re
import struct
import subprocess
import sys
import textwrap
import time
from pathlib import Path

import pytest

from nvs_testlib import FAKE_DIR, ORACLE, ROOT, Daemon, fake_env, preload

MiB = 1 << 20


def spawn(sock_dir, tmp_path, idx, mib, seconds, nbuf=3, idle=0.0, total_mib=400, extra=None):
    env = fake_env(total_mib=total_mib, ledger=tmp_path / "ledger",
                   extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_BATCH_MIB": 32,
                          "NVSHARE_DEBUG": 1, "NVSHARE_SOCK_DIR": sock_dir, "NVSHARE_POOL_GIB": 1,
                          "NVSHARE_STATS_FILE": tmp_path / f"stats{idx}.jsonl", **(extra or {})})
    env["LD_PRELOAD"] = preload("ours")
    return subprocess.Popen([str(ORACLE / "driver_app"), str(mib), str(seconds), str(idx), str(nbuf), str(idle)],
                            env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)


def finish(procs, timeout=120):
    res = []
    for p in procs:
        out, err = p.communicate(timeout=timeout)
        res.append((p.returncode, out, err))
        assert p.returncode == 0 and "RESULT PASS" in out, out + err[-2500:]
    return res


def note_retry(test, what):
    """Timing-dependent tests repeat a run that did not go to plan; how often that happens on a box is worth
    knowing (NVS_TEST_RETRY_LOG=<file>)."""
    path = os.environ.get("NVS_TEST_RETRY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(f"{time.time():.0f} {test} {what}\n")


def stats(tmp_path, idx):
    import json
    f = tmp_path / f"stats{idx}.jsonl"
    return [json.loads(l) for l in f.read_text().splitlines()] if f.exists() else []


def test_need_based_eviction_moves_only_what_the_next_client_needs(artefacts, sock_dir, tmp_path):
    # 400 MiB "HBM", two clients of 240 MiB: 1.2x oversubscribed; only ~80 MiB + margin has to move.
    # The claim is about hand-offs that go to plan.  On a loaded box a fetch may see no HBM come back for
    # 300 ms and press: the other client then frees at least 8 GiB (all of this "GPU") as a favour, and the
    # evictions around it say nothing about the need-based amount -- such a run is repeated, not judged.
    diag = []
    for attempt in range(5):
        run = tmp_path / f"run{attempt}"
        run.mkdir()
        d = Daemon("ours", sock_dir, log_path=run / "sched.log")
        try:
            d.ctl("-T", "1")
            # (the fake driver's "scan kernel" hashes 240 MiB on this CPU in about the 300 ms a waiting fetch watches
            # free HBM not growing before it presses: which side of that a run lands on is the load of the box)
            res = finish([spawn(sock_dir, run, i, 80, 6.0) for i in (1, 2)])
        finally:
            d.stop()
        ev = {i: [r for r in stats(run, i) if r["op"] == "evict"] for i in (1, 2)}
        pressed = any(r.get("favour") for i in ev for r in ev[i])
        if pressed or any(len(ev[i]) < 2 for i in ev):
            diag.append({i: [(r["bytes"] >> 20, r.get("favour")) for r in ev[i]] for i in ev})
            note_retry("need_based", diag[-1])
            continue
        for i in (1, 2):
            steady = ev[i][1:]                                # the first hand-off may have to make room for everything
            moved = [r["bytes"] + r["elided_bytes"] for r in steady]
            assert all(m < 240 * MiB for m in moved), [m >> 20 for m in moved]
            assert min(moved) <= 120 * MiB
        assert any(re.search(r"Received DROP_LOCK w1n\d+", err) for _, _, err in res)
        return
    pytest.fail(f"no run without memory-pressure favours in 5 attempts: {diag}")


def test_evict_all_policy_is_still_available(artefacts, sock_dir, tmp_path):
    d = Daemon("ours", sock_dir)
    try:
        d.ctl("-T", "1")
        finish([spawn(sock_dir, tmp_path, i, 80, 4.0, extra={"NVSHARE_EVICT_POLICY": "all"}) for i in (1, 2)])
    finally:
        d.stop()
    for i in (1, 2):
        ev = [r for r in stats(tmp_path, i) if r["op"] == "evict"]
        # everything leaves HBM every time; what has not changed since its copy was written is not copied again
        assert ev and all(r["bytes"] + r["elided_bytes"] + r["clean_bytes"] == 240 * MiB for r in ev)


def test_solo_client_keeps_its_working_set(artefacts, sock_dir, tmp_path):
    """The daemon drops the lock every TQ even when nobody waits (reference
    behaviour); with the "w0" hint our client releases the lock but keeps its
    slabs, so a solo client never pays for a hand-off."""
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "1")
        res = finish([spawn(sock_dir, tmp_path, 1, 80, 4.0)])
    finally:
        d.stop()
    assert d.read_log().count("Sent DROP_LOCK") >= 2
    assert [r for r in stats(tmp_path, 1) if r["op"] == "evict"] == []
    assert "Received DROP_LOCK w0n0" in res[0][2]


def test_pressure_evicts_an_idle_resident_client(artefacts, sock_dir, tmp_path):
    """A goes idle holding its memory (lazy release).  B arrives and cannot map:
    its pressure message reaches A through the daemon, A evicts, B proceeds; A
    later fetches everything back and verifies."""
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "30")
        a = spawn(sock_dir, tmp_path, 1, 80, 1.0, idle=9.0)          # 240 MiB of 400, then idle (releases after 5 s)
        time.sleep(7.0)
        b = spawn(sock_dir, tmp_path, 2, 80, 2.0)                     # needs 240 MiB: only ~160 are free
        res = finish([a, b])
    finally:
        d.stop()
    assert "Releasing the lock early due to inactivity" in res[0][2]
    assert re.search(r"Received DROP_LOCK e\d+", res[0][2])           # the forwarded pressure
    assert re.search(r"Sent REQ_LOCK p\d+", res[1][2])
    assert [r for r in stats(tmp_path, 1) if r["op"] == "evict"]


def test_reference_daemon_gets_the_conservative_policy(artefacts, default_sock_lock, tmp_path, have_reference):
    if not have_reference:
        pytest.skip("compiled reference not available")
    d = Daemon("reference", default_sock_lock)
    try:
        d.ctl("-T", "1")
        procs = []
        for i in (1, 2):
            env = fake_env(total_mib=400, ledger=tmp_path / "ledger",
                           extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_DEBUG": 1,
                                  "NVSHARE_POOL_GIB": 1, "NVSHARE_STATS_FILE": tmp_path / f"stats{i}.jsonl"})
            env["LD_PRELOAD"] = preload("ours")
            env["NVSHARE_SOCK_DIR"] = str(default_sock_lock)
            procs.append(subprocess.Popen([str(ORACLE / "driver_app"), "80", "4", str(i), "3"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        finish(procs)
    finally:
        d.stop()
    for i in (1, 2):     # no capability marker in the register reply -> everything is evicted on every release
        ev = [r for r in stats(tmp_path, i) if r["op"] == "evict"]
        assert ev and all(r["bytes"] + r["elided_bytes"] + r["clean_bytes"] == 240 * MiB for r in ev)


def pool_files():
    return sorted(Path("/dev/shm").glob("nvshare-pool-*"))


def test_shared_pool_lifecycle(artefacts, sock_dir, tmp_path):
    before = set(pool_files())
    d = Daemon("ours", sock_dir)
    try:
        d.ctl("-T", "1")
        procs = [spawn(sock_dir, tmp_path, i, 80, 4.0) for i in (1, 2)]
        time.sleep(3.0)
        mine = set(pool_files()) - before
        assert len(mine) == 1                                          # ONE backing file for both clients
        hdr = mine.copy().pop().open("rb").read(32)
        magic, version, window_slabs, capacity, used = struct.unpack("<QIIQQ", hdr)
        assert magic == 0x6e767368504f4f4c and version == 3 and window_slabs == 32 and capacity == 512
        finish(procs)
        res_used = struct.unpack("<QIIQQ", mine.copy().pop().open("rb").read(32))[4]
        assert res_used == 0                                           # everything handed back
    finally:
        d.stop()
    time.sleep(0.2)
    assert set(pool_files()) - before == set()                         # the daemon removes it on exit


def test_private_pool_on_request(artefacts, sock_dir, tmp_path):
    before = set(pool_files())
    d = Daemon("ours", sock_dir)
    try:
        d.ctl("-T", "1")
        procs = [spawn(sock_dir, tmp_path, i, 80, 3.0, extra={"NVSHARE_POOL": "private"}) for i in (1, 2)]
        time.sleep(1.5)
        assert set(pool_files()) - before == set()
        finish(procs)
    finally:
        d.stop()


def test_units_of_a_dead_client_are_reclaimed(artefacts, tmp_path):
    pool = tmp_path / "pool"
    code = textwrap.dedent(f"""
        import ctypes as C, os, sys
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        e = E.Engine(chunk_bytes=8 << 20, host_arena_bytes=64 << 20, shared_pool_path={str(pool)!r},
                     shared_pool_bytes=1 << 30)
        p = e.alloc(48 << 20); e.fetch_all(); e.pattern_fill(p, (48 << 20) // 8, seed=3); e.evict(0)
        print("USED", e.stats()["host_pool_used"] >> 20, flush=True)
        if sys.argv[1] == "die":
            os._exit(0)                       # no cleanup: the units stay marked with this pid
        e.fetch_all(); assert e.pattern_verify(p, (48 << 20) // 8, seed=3) == 0
        e.free(p); e.close()
    """)
    def used():
        return struct.unpack("<QIIQQ", pool.open("rb").read(32))[4]
    r = subprocess.run([sys.executable, "-c", code, "die"], capture_output=True, text=True, timeout=60)
    assert "USED 48" in r.stdout, r.stdout + r.stderr
    assert used() == 24                                                # 24 slabs leaked by the dead client
    r = subprocess.run([sys.executable, "-c", code, "live"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "USED 48" in r.stdout, r.stdout + r.stderr
    assert used() == 0                                                 # reclaimed at attach, then used and returned


def test_units_of_a_client_that_dies_later_are_reclaimed_on_exhaustion(artefacts, tmp_path):
    """The survivor is already attached when the other client dies holding most of
    the pool: its next eviction finds the pool full, reaps the dead owner's units
    and carries on instead of timing out."""
    pool = tmp_path / "pool"
    code = textwrap.dedent(f"""
        import ctypes as C, os, sys, time
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        MiB = 1 << 20
        e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, shared_pool_path={str(pool)!r},
                     shared_pool_bytes=64 * MiB, oom_wait_ms=5000, elide_constant=0, prepin=0)
        role, flag = sys.argv[1], sys.argv[2]
        p = e.alloc(48 * MiB); e.fetch_all(); e.pattern_fill(p, 48 * MiB // 8, seed=5)
        if role == "victim":
            e.evict(0); open(flag, "w").close(); os._exit(0)      # dies holding 48 of the 64 MiB
        while not os.path.exists(flag):
            time.sleep(0.01)
        time.sleep(0.2)
        e.evict(0)
        e.fetch_all(); print("BAD", e.pattern_verify(p, 48 * MiB // 8, seed=5), flush=True)
        e.free(p); e.close()
    """)
    flag = tmp_path / "victim_done"
    survivor = subprocess.Popen([sys.executable, "-c", code, "survivor", str(flag)], stdout=subprocess.PIPE,
                                stderr=subprocess.PIPE, text=True)
    time.sleep(1.0)                                                    # the survivor has attached (or created) by now
    v = subprocess.run([sys.executable, "-c", code, "victim", str(flag)], capture_output=True, text=True, timeout=60)
    assert v.returncode == 0, v.stderr
    out, err = survivor.communicate(timeout=60)
    assert survivor.returncode == 0 and "BAD 0" in out, out + err
    assert struct.unpack("<QIIQQ", pool.open("rb").read(32))[4] == 0


def test_pool_pages_are_placed_from_the_gpus_cpus(artefacts, tmp_path):
    """engine.c numa_init: the threads that populate pinned backing memory are confined
    to the CPUs next to the GPU (here forced with NVSHARE_NUMA_CPULIST, on the box read
    from sysfs), the caller's own affinity is restored, and the stats file says where
    the pages went."""
    import json
    import os
    if len(os.sched_getaffinity(0)) < 2:
        pytest.skip("needs two CPUs to tell 'near' from 'allowed'")
    near = sorted(os.sched_getaffinity(0))[0]
    pool, stats = tmp_path / "pool", tmp_path / "stats.jsonl"
    code = textwrap.dedent(f"""
        import ctypes as C, os, sys
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        before = os.sched_getaffinity(0)
        e = E.Engine(chunk_bytes=8 << 20, host_arena_bytes=64 << 20, shared_pool_path={str(pool)!r},
                     shared_pool_bytes=256 << 20, stats_path={str(stats)!r}, prepin=0)
        p = e.alloc(48 << 20); e.fetch_all(); e.pattern_fill(p, (48 << 20) // 8, seed=3); e.evict(0)
        assert os.sched_getaffinity(0) == before, "the caller's affinity was not restored"
        e.fetch_all(); assert e.pattern_verify(p, (48 << 20) // 8, seed=3) == 0
        e.free(p); e.close()
        print("OK")
    """)
    env = dict(os.environ, NVSHARE_NUMA="1", NVSHARE_NUMA_CPULIST=str(near), NVSHARE_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=60)
    assert "OK" in r.stdout, r.stdout + r.stderr
    assert "placed from 1 of" in r.stderr
    pins = [json.loads(l) for l in stats.read_text().splitlines() if '"op":"pin"' in l]
    assert pins and pins[0]["near_cpus"] == 1 and sum(pins[0]["pages_per_node"]) > 0
    env.pop("NVSHARE_NUMA")                                # opt-in: off by default
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=60)
    assert "OK" in r.stdout and "placed from" not in r.stderr


def test_background_precleaning_makes_the_first_handoff_cheap(artefacts, sock_dir, tmp_path):
    """SURVEY 8f rank 3 / VERDICT r1 #3: while a client holds the lock its resident chunks are written back
    in the background (fused copy + hash); what has not changed again by the hand-off is not copied then.
    Whether a background copy is still valid at the hand-off depends on WHEN it was taken: on a loaded box the
    application (whose "kernels" run on this CPU) may still be filling its buffers when the pre-cleaner makes
    its one pass of the residency, and every copy is stale.  The deterministic version of the claim is
    test_engine_fake.py's C-ABI test; this one is about the whole stack and gets five tries at good timing."""
    seen = []
    for attempt in range(5):
        run = tmp_path / f"run{attempt}"
        run.mkdir()
        d = Daemon("ours", sock_dir, log_path=run / "sched.log")
        try:
            d.ctl("-T", "3")
            a = spawn(sock_dir, run, 1, 80, 9.0, extra={"NVSHARE_EVICT_POLICY": "all"})
            time.sleep(2.0)                               # A alone for a while: its buffers settle and get pre-cleaned
            b = spawn(sock_dir, run, 2, 80, 6.0, extra={"NVSHARE_EVICT_POLICY": "all"})
            finish([a, b])
        finally:
            d.stop()
        recs = stats(run, 1)
        pre = sum(r["bytes"] for r in recs if r["op"] == "preclean")
        first_evict = next(r for r in recs if r["op"] == "evict")
        seen.append((pre >> 20, first_evict["clean_bytes"] >> 20))
        # two of A's three buffers are not written any more once the payload has gone round; the first
        # eviction finds their background copies still valid.  Without the pre-cleaner NOTHING is clean at a
        # first eviction, so one slab is proof enough; how many of the copies were taken after the buffers had
        # settled (160 MiB when all were) is a race between the application's start-up and the pre-cleaner's
        # one pass per residency -- in the middle of the whole suite usually 6-40 MiB
        if pre >= 160 * MiB and first_evict["clean_bytes"] >= 2 * MiB:       # one slab
            return
        note_retry("preclean", seen[-1])
    pytest.fail(f"(pre-cleaned MiB, clean MiB at the first eviction) per attempt: {seen}")


def test_precleaning_can_be_turned_off(artefacts, sock_dir, tmp_path):
    d = Daemon("ours", sock_dir)
    try:
        d.ctl("-T", "2")
        finish([spawn(sock_dir, tmp_path, i, 80, 5.0, extra={"NVSHARE_PRECLEAN": 0}) for i in (1, 2)])
    finally:
        d.stop()
    assert not [r for i in (1, 2) for r in stats(tmp_path, i) if r["op"] == "preclean"]
