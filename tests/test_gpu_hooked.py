"""LD_PRELOAD boundary on a real H100: unmodified PyTorch workloads
(nvshare_b200/workloads.py, the restated tests/pytorch-add.py and
tests/tf-matmul.py) run under OUR libnvshare.so + nvshare-scheduler, results
checked exactly; plus a genuinely oversubscribed pair made possible on a small
footprint by a ballast process that occupies most of the HBM."""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

import pytest

from nvs_testlib import ROOT, Daemon, preload

pytestmark = pytest.mark.gpu


def client_cmd(kind, n, seconds, pattern, log, tag):
    return [sys.executable, "-m", "nvshare_b200.workloads", "--kind", kind, "--n", str(n), "--iters", "1000000",
            "--seconds", str(seconds), "--pattern", pattern, "--log", str(log), "--tag", tag]


def run_pair(tmp_path, kind, n, seconds, pattern, tq, extra_env=None):
    sock_dir = tmp_path / "nvs"
    sock_dir.mkdir(exist_ok=True)
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", str(tq))
        procs = []
        for i in (1, 2):
            env = dict(os.environ, LD_PRELOAD=preload("ours"), NVSHARE_SOCK_DIR=str(sock_dir),
                       NVSHARE_STATS_FILE=str(tmp_path / f"stats{i}.jsonl"), PYTHONPATH=str(ROOT))
            env.update(extra_env or {})
            procs.append(subprocess.Popen(client_cmd(kind, n, seconds, pattern, tmp_path / f"c{i}.jsonl", f"c{i}"),
                                          env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=900) for p in procs]
        return d.read_log(), [(p.returncode, o, e) for p, (o, e) in zip(procs, outs)]
    finally:
        d.stop()


def stats(tmp_path, i):
    p = tmp_path / f"stats{i}.jsonl"
    return [json.loads(l) for l in p.read_text().splitlines()] if p.exists() else []


def test_add_two_clients_exact(artefacts, tmp_path):
    """BASELINE config #2 at small scale: fp32 add, position-dependent inputs, bit-exact."""
    # evict-all policy: both working sets would fit side by side at this size, so force the swap
    log, res = run_pair(tmp_path, "add", 12000, 8, "pos", tq=2, extra_env={"NVSHARE_EVICT_POLICY": "all"})
    for rc, out, err in res:
        assert rc == 0 and out.startswith("PASS"), out + err[-3000:]
    assert log.count("Sent DROP_LOCK") >= 2
    for i in (1, 2):
        ops = [r["op"] for r in stats(tmp_path, i)]
        assert "evict" in ops and "fetch" in ops            # the engine really swapped under the hook


def test_no_swap_when_everything_fits(artefacts, tmp_path):
    """Default (need-based) policy: two small clients fit in HBM together, so hand-offs move nothing."""
    log, res = run_pair(tmp_path, "add", 8000, 5, "ones", tq=1)
    for rc, out, err in res:
        assert rc == 0 and out.startswith("PASS"), out + err[-3000:]
    assert log.count("Sent DROP_LOCK") >= 3
    for i in (1, 2):
        assert [r for r in stats(tmp_path, i) if r["op"] == "evict"] == []


@pytest.mark.parametrize("pattern", ["ones", "pos"])
def test_matmul_two_clients_within_tolerance(artefacts, tmp_path, pattern):
    """BASELINE config #3 restated with torch.matmul (three n x n blocks, product in place, TF32 like
    TensorFlow 2.7): ones x ones == n, ones x pos == exact column sums, within 1e-5 relative -- with
    every hand-off FORCED to swap (both clients would fit side by side at this size), and the swap
    asserted.  "ones": operands are same-filled and described, not moved; "pos": they really move."""
    # "pos" counts the bytes the EVICTIONS copy, so the background pre-cleaner stays out of it: it would write the
    # operand and the (always identical) product back during the quantum and leave the evictions nothing to copy
    env = {"NVSHARE_EVICT_POLICY": "all"}
    if pattern == "pos":
        env["NVSHARE_PRECLEAN"] = "0"
    log, res = run_pair(tmp_path, "matmul", 8192, 8, pattern, tq=2, extra_env=env)
    for rc, out, err in res:
        assert rc == 0 and out.startswith("PASS"), out + err[-3000:]
    assert log.count("Sent DROP_LOCK") >= 2
    for i in (1, 2):
        recs = stats(tmp_path, i)
        ev = [r for r in recs if r["op"] == "evict"]
        assert ev and any(r["op"] == "fetch" for r in recs)            # the engine really swapped under the hook
        moved = sum(r["bytes"] for r in ev)
        if pattern == "ones":
            assert sum(r["elided_bytes"] for r in ev) > 0
        else:
            assert moved >= 2 * 8192 * 8192 * 4                        # the operand and the product crossed the link


def test_same_workload_under_the_reference_library_and_ours(artefacts, tmp_path, have_reference, request):
    """Ours and -- where it can run -- the reference's libnvshare.so + nvshare-scheduler (oracle/_ref,
    unmodified: cuMemAllocManaged and UVM faults) run the same seeded workloads on the same GPU; each
    verifies its own results and prints checksums of its output tensor, which must be identical to
    those of the un-hooked application (tests/golden/workload_checksums.json, make_golden.py)."""
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    from make_golden import CHECKSUM_WORKLOADS
    gold = json.loads((ROOT / "tests" / "golden" / "workload_checksums.json").read_text())
    sums = {}
    for arm in (("reference", "ours") if have_reference else ("ours",)):
        sock_dir = request.getfixturevalue("default_sock_lock") if arm == "reference" else tmp_path / "nvs"
        sock_dir.mkdir(exist_ok=True)
        d = Daemon(arm, sock_dir, log_path=tmp_path / f"sched_{arm}.log")
        try:
            d.ctl("-T", "2", impl=arm)
            procs = []
            for i, (kind, n) in enumerate(CHECKSUM_WORKLOADS):
                env = dict(os.environ, LD_PRELOAD=preload(arm), PYTHONPATH=str(ROOT), NVSHARE_EVICT_POLICY="all")
                if arm == "ours":
                    env["NVSHARE_SOCK_DIR"] = str(sock_dir)
                procs.append(subprocess.Popen(client_cmd(kind, n, 6, "pos", tmp_path / f"{arm}{i}.jsonl", f"{arm}{i}"),
                                              env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
            for i, p in enumerate(procs):
                out, err = p.communicate(timeout=900)
                assert p.returncode == 0 and out.startswith("PASS"), arm + out + err[-3000:]
                summary = json.loads(out.splitlines()[0].split(" ", 1)[1])
                sums[(arm, i)] = [summary["z_sum"], summary["z_wsum"]]
        finally:
            d.stop()
    for (arm, i), got in sums.items():
        kind, n = CHECKSUM_WORKLOADS[i]
        assert got == gold[f"{kind}_{n}"], (arm, kind, got)


def test_oversubscribed_pair_with_ballast(artefacts, tmp_path):
    """Real oversubscription: a ballast process pins most of the HBM, leaving room
    for ~1.4 client footprints; two clients then alternate and must stay exact."""
    import torch
    free, total = torch.cuda.mem_get_info()
    footprint = 4 * 4 * 16000 * 16000                       # four n^2 fp32 blocks, ~4.1 GB
    keep = int(footprint * 1.45) + (3 << 30)                 # what the pair may use (+ contexts)
    ballast_bytes = free - keep
    code = ("import torch,sys,time; b=torch.empty(%d,dtype=torch.uint8,device='cuda'); torch.cuda.synchronize();"
            "print('BALLAST',flush=True); time.sleep(10000)" % ballast_bytes)
    ballast = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, text=True)
    try:
        assert "BALLAST" in ballast.stdout.readline()
        log, res = run_pair(tmp_path, "add", 16000, 10, "pos", tq=2)
    finally:
        ballast.kill()
        ballast.wait()
    for rc, out, err in res:
        assert rc == 0 and out.startswith("PASS"), out + err[-3000:]
    waits = [r.get("wait_ms", 0) for i in (1, 2) for r in stats(tmp_path, i) if r["op"] == "fetch"]
    assert len(waits) >= 4


def test_uvm_mode_add(artefacts, tmp_path):
    log, res = run_pair(tmp_path, "add", 8000, 4, "ones", tq=2, extra_env={"NVSHARE_ENGINE": "uvm"})
    for rc, out, err in res:
        assert rc == 0 and out.startswith("PASS"), out + err[-3000:]


def test_loading_client_does_not_take_the_gpu(artefacts, tmp_path):
    """SURVEY 8f rank 3 with the real CUDA runtime: while client A computes inside
    a 30 s quantum, client B (tests/apps/torch_loader.py) allocates, uploads 2 x
    256 MiB and reads them back WITHOUT asking for the lock -- the copies are
    served from the pinned-host backing copy -- and only its first kernel waits."""
    sock_dir = tmp_path / "nvs"
    sock_dir.mkdir()
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", "30")
        env = dict(os.environ, LD_PRELOAD=preload("ours"), NVSHARE_SOCK_DIR=str(sock_dir), PYTHONPATH=str(ROOT),
                   NVSHARE_DEBUG="1")
        a = subprocess.Popen(client_cmd("add", 8000, 25, "ones", tmp_path / "a.jsonl", "a"), env=env, cwd=ROOT,
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        deadline = time.time() + 120
        while "Sent LOCK_OK" not in d.read_log():          # A holds the lock
            assert time.time() < deadline and a.poll() is None
            time.sleep(0.2)
        b = subprocess.run([sys.executable, str(ROOT / "tests" / "apps" / "torch_loader.py")], env=env, cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        out_a, err_a = a.communicate(timeout=600)
    finally:
        d.stop()
    assert a.returncode == 0 and out_a.startswith("PASS"), out_a + err_a[-3000:]
    assert b.returncode == 0 and "RESULT PASS" in b.stdout, b.stdout + b.stderr[-3000:]
    load = [l for l in b.stdout.splitlines() if l.startswith("LOAD_DONE")][0].split()
    assert load[2] == "True" and float(load[1]) < 6.0, b.stdout                 # far inside A's 25 s of work
    err = b.stderr
    assert err.count("served from the backing copy") >= 4
    assert err.index("served from the backing copy") < err.index("Sent REQ_LOCK")   # the lock was asked for afterwards


def _pair_of(tmp_path, argv_of, tq=1, extra_env=None, timeout=600):
    sock_dir = tmp_path / "nvs"
    sock_dir.mkdir(exist_ok=True)
    d = Daemon("ours", sock_dir, log_path=tmp_path / "sched.log")
    try:
        d.ctl("-T", str(tq))
        procs = []
        for i in (1, 2):
            env = dict(os.environ, LD_PRELOAD=preload("ours"), NVSHARE_SOCK_DIR=str(sock_dir), PYTHONPATH=str(ROOT),
                       NVSHARE_EVICT_POLICY="all", NVSHARE_STATS_FILE=str(tmp_path / f"stats{i}.jsonl"))
            env.update(extra_env or {})
            procs.append(subprocess.Popen(argv_of(i), env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=timeout) for p in procs]
        return d.read_log(), [(p.returncode, o, e) for p, (o, e) in zip(procs, outs)]
    finally:
        d.stop()


def _assert_swapped(tmp_path, log, res):
    for rc, out, err in res:
        assert rc == 0 and "RESULT PASS" in out, out + err[-3000:]
    assert log.count("Sent DROP_LOCK") >= 2
    for i in (1, 2):
        ops = [r["op"] for r in stats(tmp_path, i)]
        assert "evict" in ops and "fetch" in ops


def test_cuda_graph_replays_through_forced_swaps(artefacts, tmp_path):
    """SURVEY 8f rank 2: cuGraphLaunch is gated (the reference lets it through), the capture itself is
    not disturbed by the launch hook's synchronisation window, and the memory the graph's nodes
    point at is unmapped and re-mapped under it between replays."""
    log, res = _pair_of(tmp_path, lambda i: [sys.executable, str(ROOT / "tests" / "apps" / "graph_app.py"), "4096", "8"])
    _assert_swapped(tmp_path, log, res)


def test_cooperative_launches_through_forced_swaps(artefacts, tmp_path):
    """cuLaunchCooperativeKernel (grid-wide sync) is gated too; runtime-API application, exact 64-bit check."""
    from nvs_testlib import ORACLE
    app = ORACLE / "coop_app"
    if not app.exists():
        pytest.skip("oracle/_ref/coop_app not built (needs nvcc at build time)")
    log, res = _pair_of(tmp_path, lambda i: [str(app), "512", "8", str(i)])
    _assert_swapped(tmp_path, log, res)


def test_stream_ordered_allocator_backend_is_capped_and_swapped(artefacts, tmp_path):
    """PyTorch with backend:cudaMallocAsync: every tensor comes from cuMemAllocAsync / cuMemFreeAsync, which
    the reference neither charges to the cap nor makes swappable.  Here they go through the swap engine."""
    log, res = run_pair(tmp_path, "add", 12000, 8, "pos", tq=2,
                        extra_env={"NVSHARE_EVICT_POLICY": "all", "PYTORCH_CUDA_ALLOC_CONF": "backend:cudaMallocAsync"})
    for rc, out, err in res:
        assert rc == 0 and out.startswith("PASS"), out + err[-3000:]
    for i in (1, 2):
        recs = stats(tmp_path, i)
        assert sum(r["bytes"] + r.get("clean_bytes", 0) for r in recs if r["op"] == "evict") >= 3 * 12000 * 12000 * 4
