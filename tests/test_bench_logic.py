"""bench.py's host-side decisions, CPU only: geometry of the BASELINE
configuration and the host-memory-aware scale selection."""
from __future__ import annotations

import importlib.util
import math
import types
from pathlib import Path

from nvs_testlib import ROOT


def load_bench(shm_bytes=1 << 40):
    """bench.py as a module, with /dev/shm reporting `shm_bytes` of free space."""
    spec = importlib.util.spec_from_file_location("bench_module", ROOT / "bench.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    real_os = m.os

    class FakeOS:
        def __getattr__(self, name):
            return getattr(real_os, name)

        @staticmethod
        def statvfs(path):
            return types.SimpleNamespace(f_bavail=shm_bytes // 4096, f_frsize=4096)

    m.os = FakeOS()
    return m


def pick(b, impl="ours", forced=0.0, world=1):
    return b.pick_fraction(impl, 2, 1.5, HBM, forced, world)


HBM = 85_017_493_504           # what cuMemGetInfo reports on an H100 80GB HBM3


def test_full_scale_fits_for_ours_but_not_for_the_reference(monkeypatch):
    b = load_bench()
    monkeypatch.setattr(b, "host_memory_budget", lambda: 110_000_000_000)     # a box with a 110 GB memory cgroup
    assert pick(b, "ours") == (1.0, None)
    frac, note = pick(b, "reference")
    assert 0.5 <= frac <= 0.65 and "host RAM budget" in note
    # an explicit fraction is never overridden
    assert pick(b, "reference", forced=0.25) == (0.25, None)
    # the peer tier keeps next to nothing on the host
    assert pick(b, "ours", world=2) == (1.0, None)


def test_no_limit_means_full_scale(monkeypatch):
    b = load_bench()
    monkeypatch.setattr(b, "host_memory_budget", lambda: None)
    assert pick(b, "reference") == (1.0, None)
    monkeypatch.setattr(b, "host_memory_budget", lambda: 2_000_000_000_000)
    assert pick(b, "reference") == (1.0, None)


def test_host_memory_model():
    b = load_bench()
    f = 0.75 * HBM
    # the reference keeps every client's pages on the host; ours only what is swapped out (+ pinned windows ahead)
    assert b.host_memory_needed("reference", 2, f, HBM) > 2 * f
    assert b.host_memory_needed("ours", 2, f, HBM) < 2 / 3 * b.host_memory_needed("reference", 2, f, HBM)
    assert b.host_memory_needed("ours", 2, 0.4 * HBM, HBM) < 40e9          # fits: nothing to swap


def test_small_dev_shm_means_private_pools(monkeypatch):
    # docker's default 64 MiB /dev/shm: every client pins its own arenas, which no longer fits at full scale
    b = load_bench(shm_bytes=64 << 20)
    f = 0.75 * HBM
    assert b.host_memory_needed("ours", 2, f, HBM) > 2 * (2 * f - HBM)
    monkeypatch.setattr(b, "host_memory_budget", lambda: 110_000_000_000)
    frac, note = pick(b, "ours")
    assert frac < 1.0 and note


def test_baseline_geometry():
    # four live n^2 fp32 blocks per client (x, y, z and the allocator's cached block): SURVEY 8d
    n = int(math.floor(math.sqrt(1.5 * HBM / 2 / 16)))
    assert n == 63128
    assert abs(4 * 4 * n * n - 0.75 * HBM) / (0.75 * HBM) < 1e-4


def test_client_specs_reach_the_footprint():
    b = load_bench()
    spec, fp = b.make_spec("add", "pos", 0.75 * HBM)
    assert spec["n"] == 63128 and fp <= 0.75 * HBM
    spec, fp = b.make_spec("matmul", "pos", 0.75 * HBM)          # three blocks like the reference's TF graph
    assert spec["n"] == int(math.floor(math.sqrt(0.75 * HBM / 12))) and abs(fp - 0.75 * HBM) / HBM < 1e-4
    spec, fp = b.make_spec("llama", "pos", 0.75 * HBM)
    kv = spec["batch"] * spec["context"] * (1 << 20)               # 7B geometry, fp32: 1 MiB of KV per token
    assert spec["size"] == "7b" and 27e9 + kv < fp and fp - (27e9 + kv) < 16e9
    spec, fp = b.make_spec("resnet", "pos", 0.95 * HBM)
    assert spec["target_bytes"] == int(0.95 * HBM)


def test_algorithmic_bytes_are_independent_of_the_number_of_clients():
    # what must come in per hand-off: the arriving client's footprint minus the HBM the holder leaves free
    f = 0.75 * HBM
    assert abs(max(min(f, 2 * f - HBM), 0) - 0.5 * HBM) < 1


def test_sub_runs_live_inside_the_time_budget(monkeypatch):
    """The driver gives every `bench.py --gpus N` run a fixed time; the sub-runs (same-scale pair, configs #4/#5)
    only get what the headline left, and say so when they were skipped."""
    b = load_bench()
    calls = []

    def fake_run(impl, kind, *a, **kw):
        calls.append((kind, kw.get("time_limit_s")))
        return {"kind": kind, "impl": impl, "verified": True, "spec": {}}
    monkeypatch.setattr(b, "run_experiment", fake_run)
    monkeypatch.setattr(b, "pick_fraction", lambda impl, *a, **k: (0.6, "note") if impl == "reference" else (1.0, None))
    a = types.SimpleNamespace(kind="add", pattern="pos", clients=2, oversub=1.5, tq=10, warmup=5, steps=20)
    # plenty of time: N=1 runs the same-scale pair, N=2 config #4, N=8 config #5, N=4 nothing
    for world, want in ((1, ["add"]), (2, ["resnet"]), (8, ["llama"]), (4, [])):
        calls.clear()
        line = {}
        b.extras(a, line, {}, world, HBM, 1.0, Path("/tmp/x"), b.time.time())
        assert [k for k, _ in calls] == want
        assert all(0 < lim <= b.TOTAL_BUDGET_S for _, lim in calls)
    # the headline used the budget up: nothing is started, and the line says why
    calls.clear()
    line = {}
    b.extras(a, line, {}, 2, HBM, 1.0, Path("/tmp/x"), b.time.time() - (b.TOTAL_BUDGET_S - 100))
    assert calls == [] and "skipped" in line["configs"]["config4_resnet50_train_x2_2xHBM_peer_tier"]
    line = {}
    b.extras(a, line, {}, 1, HBM, 1.0, Path("/tmp/x"), b.time.time() - (b.TOTAL_BUDGET_S - 100))
    assert calls == [] and "skipped" in line["same_scale"]


def test_reference_arm_probes_load_nothing_of_ours(monkeypatch):
    """`bench.py --impl reference` must not touch our kernels or engine anywhere, its probe child included."""
    b = load_bench()
    seen = {}

    def fake_run(cmd, **kw):
        seen["env"] = kw["env"]
        return types.SimpleNamespace(returncode=0, stdout='PROBE {"hbm_total": 1, "link": {"h2d": 1, "d2h": 1}}\n', stderr="")
    monkeypatch.setattr(b.subprocess, "run", fake_run)
    try:
        b.run_probes(kernels=False)
    except Exception:
        pass                      # the reply format is not what is being tested
    assert seen["env"]["NVS_BENCH_PROBE_KERNELS"] == "0"
    try:
        b.run_probes()
    except Exception:
        pass
    assert seen["env"]["NVS_BENCH_PROBE_KERNELS"] == "1"
    src = (ROOT / "bench.py").read_text()
    assert 'run_probes(kernels=args.impl == "ours")' in src


def test_run_experiment_post_processing_on_synthetic_records(tmp_path, monkeypatch):
    """Everything bench.py does around a run -- the time-limit split of a sub-run, the analysis, the `device` record
    from the engines' stats lines, the roofline objects -- executed on CPU over synthetic client timelines and
    engine records (the clients themselves need a GPU)."""
    import json
    b = load_bench()
    tq, stall, tau = 1.0, 0.4, 0.02
    t, who, iters, recs = 1000.0, 0, {0: [], 1: []}, {0: [], 1: []}
    for _ in range(12):                                    # 12 quanta = 11 hand-offs
        t += stall
        recs[who].append({"op": "fetch", "t": t, "bytes": 50 << 30, "copy_ms": 900.0, "host_bytes": 50 << 30, "peer_bytes": 0,
                          "launches": 0, "ce_calls": 200, "map_ms": 60.0, "wait_ms": 150.0, "wall_ms": 1100.0, "elided_bytes": 0,
                          "retained_bytes": 40 << 30, "pool_used": 90 << 30})
        end = t + tq
        while t < end:
            t += tau
            iters[who].append(t)
        recs[who].append({"op": "evict", "t": t + 0.3, "bytes": 5 << 30, "copy_ms": 100.0, "host_bytes": 5 << 30, "peer_bytes": 0,
                          "launches": 3, "scan_launches": 2, "ce_calls": 20, "map_ms": 90.0, "wait_ms": 0.0, "wall_ms": 400.0,
                          "scanned_bytes": 140 << 30, "scan_ms": 24.0, "clean_bytes": 45 << 30, "elided_bytes": 0,
                          "retained_bytes": 40 << 30, "pool_used": 90 << 30})
        who ^= 1
    seen = {}

    def fake_run_clients(impl, out_dir, n, spec, seconds, tq_, extra_env=None, stop_after_handoffs=0, setup_timeout=0, **kw):
        seen.update(seconds=seconds, setup_timeout=setup_timeout, stop_after=stop_after_handoffs)
        for i in (0, 1):
            (Path(out_dir) / f"engine{i}.jsonl").write_text("".join(json.dumps(r) + "\n" for r in recs[i]))
        return [{"rc": 0, "iters": iters[i], "meta": {"summary": {"result": "PASS"}}, "out": "", "err_tail": ""} for i in (0, 1)]

    class Sampler:
        def __init__(self, *a, **k): pass
        def start(self): pass
        def stop(self, *a, **k): return {"sm_mhz": 1800.0, "sm_max_mhz": 1965.0, "reasons": []}
    monkeypatch.setattr(b.harness, "calibrate", lambda spec, out, env=None: {"tau_s": tau, "iters": 100})
    monkeypatch.setattr(b.harness, "run_clients", fake_run_clients)
    monkeypatch.setattr(b.harness, "ClockSampler", Sampler)
    exp = b.run_experiment("ours", "add", "pos", 2, 1.5, tq, 2, 4, HBM, 1.0, 1, tmp_path / "x", time_limit_s=300)
    assert "error" not in exp, exp
    # the timed part got what (2 + 4 + 2) hand-offs need, the setup the rest, and together they stay inside the limit
    assert seen["stop_after"] == 8 and seen["seconds"] >= 8 * (tq + 4) and seen["setup_timeout"] + seen["seconds"] + 20 <= 300 + 1e-6
    assert exp["verified"] and abs(exp["stall_ms_per_handoff"] - 1e3 * stall) < 60
    dev = exp["device"]
    assert dev["fetches"] >= 4 and dev["evicts"] >= 4 and dev["scan_GBps"] > 1000
    assert "gpu_ledger" not in dev                        # host tier: the engines say nothing about peers
    ratio = dev["link_bytes_over_algorithmic"]            # per transfer, not per timed step
    assert abs(ratio["in"] - (50 << 30) / exp["algorithmic_bytes_per_handoff_per_direction"]) < 1e-9
    assert abs(ratio["out"] - (5 << 30) / exp["algorithmic_bytes_per_handoff_per_direction"]) < 1e-9
    roof = b.roofline_objects(exp, {"link": {"h2d": 55.0, "d2h": 52.0}}, 1)
    assert roof["roofline"]["kernel"] == "nvs_slab_scan" and roof["roofline"]["frac"] > 0
    assert roof["roofline_link"]["fetch"]["frac"] > 0 and roof["roofline_link"]["evict"]["peak"] == 52.0
    brief = b.brief(exp)
    assert brief["verified"] and "stall_ms_per_handoff" in brief
    # peer tier: the engines' view of the cross-process GPU ledger travels with their transfer records
    for i in (0, 1):
        for r in recs[i]:
            r.update({"peer_pool_bytes": 30 << 30, "gl_tracked_peers": 1, "gl_lent": 55 << 30, "gl_my_lent": 30 << 30, "gl_refusals": 0})
    exp_p = b.run_experiment("ours", "add", "pos", 2, 1.5, tq, 2, 4, HBM, 1.0, 2, tmp_path / "y", time_limit_s=300)
    led = exp_p["device"]["gpu_ledger"]
    assert led == {"tracked_peers": 1, "lent_bytes_max": 55 << 30, "one_client_lent_bytes_max": 30 << 30,
                   "one_client_arena_bytes_max": 30 << 30, "own_claim_matches_arenas": True, "refusals": 0}
    assert b.brief(exp_p)["device"]["gpu_ledger"] == led
    roof2 = b.roofline_objects(exp, {"link": {"h2d": 55.0, "d2h": 52.0}, "peer": {"out": 781.0, "in": 780.0}}, 2)
    assert roof2["roofline"]["bound"] == "nvlink" and roof2["roofline"]["peak"] == 780.5 and "roofline_scan" in roof2


def test_the_json_line_of_both_arms_is_assembled_on_cpu(tmp_path, monkeypatch):
    """run_rank0 from probes to the finished line, with the GPU-bound pieces replaced: every key of the bench contract
    is there for our arm, and the reference arm carries its own cpu_baseline / e2e and launches nothing of ours."""
    import json
    b = load_bench()
    tq, stall, tau = 1.0, 0.4, 0.02
    t, who, iters, recs = 1000.0, 0, {0: [], 1: []}, {0: [], 1: []}
    for _ in range(12):
        t += stall
        recs[who].append({"op": "fetch", "t": t, "bytes": 50 << 30, "copy_ms": 900.0, "host_bytes": 50 << 30, "peer_bytes": 0,
                          "launches": 0, "ce_calls": 200, "map_ms": 60.0, "wait_ms": 150.0, "wall_ms": 1100.0, "elided_bytes": 0})
        end = t + tq
        while t < end:
            t += tau
            iters[who].append(t)
        recs[who].append({"op": "evict", "t": t + 0.3, "bytes": 5 << 30, "copy_ms": 100.0, "host_bytes": 5 << 30, "peer_bytes": 0,
                          "launches": 3, "scan_launches": 2, "ce_calls": 20, "map_ms": 90.0, "wait_ms": 0.0, "wall_ms": 400.0,
                          "scanned_bytes": 140 << 30, "scan_ms": 24.0, "clean_bytes": 45 << 30, "elided_bytes": 0})
        who ^= 1

    def fake_run_clients(impl, out_dir, n, spec, seconds, tq_, **kw):
        if impl == "ours":
            for i in (0, 1):
                (Path(out_dir) / f"engine{i}.jsonl").write_text("".join(json.dumps(r) + "\n" for r in recs[i]))
        return [{"rc": 0, "iters": iters[i], "meta": {"summary": {"result": "PASS"}}, "out": "", "err_tail": ""} for i in (0, 1)]

    class Sampler:
        def __init__(self, *a, **k): pass
        def start(self): pass
        def stop(self, *a, **k): return {"sm_mhz": 1800.0, "sm_max_mhz": 1965.0, "reasons": []}
    probes = []
    monkeypatch.setattr(b.harness, "calibrate", lambda spec, out, env=None: {"tau_s": tau, "iters": 100})
    monkeypatch.setattr(b.harness, "run_clients", fake_run_clients)
    monkeypatch.setattr(b.harness, "ClockSampler", Sampler)
    monkeypatch.setattr(b, "run_probes", lambda kernels=True: probes.append(kernels) or
                        {"hbm_total": HBM, "link": {"h2d": 55.0, "d2h": 52.0}, "kernels": {"scan_hash": {}} if kernels else None})
    monkeypatch.setattr(b, "cpu_baseline", lambda: {"value": 8.9, "unit": "GB/s", "cores": 1, "kind": "port", "sample": "x"})
    monkeypatch.setattr(b, "host_memory_budget", lambda: None)
    monkeypatch.setattr(b.subprocess, "Popen", None)       # nothing may be started behind the stubs' back
    for impl in ("ours", "reference"):
        if impl == "reference" and not b.harness.impl_paths("reference")["lib"].exists():
            continue
        args = types.SimpleNamespace(impl=impl, kind="add", pattern="pos", clients=2, oversub=1.5, tq=tq, warmup=2, steps=4,
                                     hbm_fraction=1.0, keep=str(tmp_path / impl), no_extras=True, gpus=1)
        line, wall = b.run_rank0(args, 1)
        json.dumps(line)                                   # serialisable
        for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                  "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "cpu_baseline", "verified"):
            assert k in line, (impl, k)
        assert line["impl"] == impl and line["verified"] and line["config"]["workload"]
        assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(line["e2e"])
        if impl == "ours":
            assert line["gpu_launches"] > 0 and line["roofline"]["kernel"] == "nvs_slab_scan" and line["cpu_baseline"]["kind"] == "port"
            assert line["e2e"]["h2d_bytes_per_step"] > 0
        else:
            assert line["gpu_launches"] == 0 and line["cpu_baseline"]["kind"] == "reference" and "roofline" not in line
            assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["value"] == line["value"]
    assert probes[0] is True and (len(probes) == 1 or probes[1] is False)
