#!/usr/bin/env python3
"""bench.py -- BASELINE.json's metric on its config:

    swap GB/s + iter/sec at 1.5x HBM oversubscription, 2 co-located clients
    (restated tests/pytorch-add.py), vs the reference's UVM page-fault path.

One STEP = one lock hand-off between the clients (the leaving client's working
set goes out, the arriving client's comes in) together with the quantum of
client compute that follows it.  W warm-up hand-offs, then exactly K timed
hand-offs, delimited on the merged per-iteration timeline of the clients
(nvshare_b200/harness.py); both arms are analysed by the same code, with the
resident iteration time tau taken from a solo, un-hooked calibration run of the
same application.

JSON line (one, from rank 0):
  value      swap GB/s measured ON THE DEVICE: payload bytes that crossed the link
             in the timed hand-offs / CUDA-event time of those transfers (both
             directions; inputs resident in HBM / pinned host memory when each
             transfer starts)
  e2e.value  the same metric END TO END through the LD_PRELOAD boundary:
             2 x algorithmic bytes per hand-off / measured stall per hand-off, as
             the unmodified PyTorch application experiences it (host<->device
             copies, map/unmap, scan, protocol and scheduling all inside)
  iter_per_s oversubscribed-client iterations per second over the timed window
  roofline   the dominant sm_90a kernel of the timed region against the measured
             peak that bounds it: at N=1 the scan/hash kernel (HBM-bound; the bytes
             themselves cross PCIe on the copy engines -- `roofline_link` has both
             directions against the link peak measured in this run); at N>1 the
             TMA slab-copy kernel against the peer-copy peak measured in this run
  cpu_baseline  oracle/nvshare_oracle.c's migration restatement (memcpy) on one
             host core, bounded sample -- reported, not a target
  same_scale (N=1) our arm once more at the HBM fraction the reference arm has to
             fall back to on this box (its UVM needs every client's footprint in
             host RAM), so that a same-configuration pair exists in one record
  configs    (N=2 / N=8) BASELINE configs #4 / #5 as verified sub-runs on the peer
             tier: ResNet-50 training x2 at ~2x HBM, 4 x Llama-7B decode at 3x

--impl reference runs the UNMODIFIED reference (oracle/_ref: its libnvshare.so
and nvshare-scheduler, i.e. cuMemAllocManaged + UVM faults) through the same
harness on the same workload.

Multi-GPU (--gpus N under torchrun): the path shards by slab, not by client:
rank 0 hosts the clients on GPU 0 and stripes their backing slabs over the
HBM of GPUs 1..N-1 (peer tier, cuMemMap of peer physical memory, no NCCL);
the other ranks only take part in the barriers.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
# nothing is written into the tree at run time (it may be read-only): no bytecode caches, here or in the clients
sys.dont_write_bytecode = True
os.environ["PYTHONDONTWRITEBYTECODE"] = "1"

from nvshare_b200 import harness  # noqa: E402

GiB = 1 << 30
MiB = 1 << 20
T_START = time.time()          # of this process: the driver's clock around the run starts about here
METRIC = "swap_GBps_at_1.5x_hbm_oversub_2_clients"


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", choices=["ours", "reference"], default="ours")
    ap.add_argument("--tq", type=int, default=0, help="scheduler time quantum in seconds (reference default: 30); "
                    "0 = 10 for add (the reference's README: \"don't set TQ < 10\"), 30 for matmul, 5 for the model configs")
    ap.add_argument("--oversub", type=float, default=0.0, help="aggregate client footprint / HBM (0 = the BASELINE value of the kind)")
    ap.add_argument("--clients", type=int, default=0)
    ap.add_argument("--kind", choices=["add", "matmul", "resnet", "llama"], default="add")
    ap.add_argument("--pattern", choices=["ones", "pos"], default="pos")
    ap.add_argument("--hbm-fraction", type=float, default=0.0,
                    help="share of the GPU's HBM the experiment may use; the rest is held by a ballast process. "
                         "1.0 = the configuration BASELINE.json names; 0 (default) = 1.0 if the host memory this "
                         "arm needs fits the box's limit, else the largest fraction that does")
    ap.add_argument("--no-extras", action="store_true", help="skip the same_scale / configs sub-runs")
    ap.add_argument("--keep", default="", help="directory to keep logs in")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="after the timed steps every client writes a fixed, seeded sample of the output it computed "
                         "in its last step and of its inputs to DIR/client<i>_{z,x,y,index}.npy (add and matmul); the "
                         "inputs follow from the arguments and the HBM fraction (--hbm-fraction pins it across boxes)")
    ap.add_argument("--probe", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump_outputs and args.kind not in ("add", "matmul"):
        ap.error("--dump-outputs is implemented for --kind add and matmul")
    return args


def dist_env():
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    return rank, world, local


# ------------------------------------------------------------------ probes --
# Run in a child process (`bench.py --probe`): the parent never creates a CUDA context on
# GPU 0 at N=1, so the clients have the whole HBM (fewer bytes per hand-off).

def measure_link_peak(torch, nbytes=2 * GiB):
    """Copy-engine H2D / D2H bandwidth with pinned memory, CUDA events: the
    roofline denominator for the host tier, measured on this box in this run."""
    dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    out = {}
    for name, (dst, src) in {"d2h": (host, dev), "h2d": (dev, host)}.items():
        best = 0.0
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dst.copy_(src, non_blocking=True)
            e1.record()
            e1.synchronize()
            best = max(best, nbytes / 1e6 / e0.elapsed_time(e1))
        out[name] = best
    del dev, host
    torch.cuda.empty_cache()
    return out


def measure_peer_peak(torch, nbytes=4 * GiB):
    """GPU 0 <-> GPU 1 over NVLink with the copy engines (one large cuMemcpyPeer each way)."""
    if torch.cuda.device_count() < 2:
        return None
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    b = torch.empty(nbytes, dtype=torch.uint8, device="cuda:1")
    out = {}
    for name, (dst, src) in {"out": (b, a), "in": (a, b)}.items():
        best = 0.0
        for _ in range(4):
            torch.cuda.synchronize(0); torch.cuda.synchronize(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.device(0):
                e0.record()
                dst.copy_(src, non_blocking=True)
                e1.record()
                e1.synchronize()
            best = max(best, nbytes / 1e6 / e0.elapsed_time(e1))
        out[name] = best
    return out


def measure_hbm_peak(torch, nbytes=4 * GiB):
    """HBM read + write traffic of b.copy_(a) device-to-device, CUDA events, best of 3: the roofline
    denominator for the HBM-bound kernels, measured on this GPU in this run."""
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b.copy_(a)
    best = 0.0
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        b.copy_(a)
        e1.record()
        e1.synchronize()
        best = max(best, 2 * nbytes / 1e6 / e0.elapsed_time(e1))
    del a, b
    torch.cuda.empty_cache()
    return best


def hbm_peak(probe):
    if probe.get("hbm_copy_GBps"):
        return probe["hbm_copy_GBps"], "b.copy_(a) device-to-device (read + write traffic) measured in this run"
    return 3350.0, "H100 SXM data sheet (HBM3), not measured in this run"


def measure_kernels(torch, peak, source, nbytes=4 * GiB):
    """The sm_90a kernels alone, through the C-ABI: the TMA slab copy device-to-device on all SMs (shows the
    link, not the kernel, bounds the NVLink/PCIe path) and the scan/hash kernel over the same bytes."""
    from nvshare_b200 import engine as E
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    src.random_(0, 255)
    descs = [(src.data_ptr() + o, dst.data_ptr() + o, 2 * MiB) for o in range(0, nbytes, 2 * MiB)]
    with E.Engine(prepin=0) as e:
        n_sms = torch.cuda.get_device_properties(0).multi_processor_count
        e.copy_slabs(descs, variant="tma", grid=n_sms)
        ms = min(e.copy_slabs(descs, variant="tma", grid=n_sms) for _ in range(3))
        ok = bool(torch.equal(src, dst))
        E.scan_slabs(e, descs, want_hash=True)
        scans = [E.scan_slabs(e, descs, want_hash=True, with_ms=True) for _ in range(3)]
        scan_ms = min(m for _, m in scans)
        same = all(a == b for a, b in zip(scans[0][0], scans[1][0]))
    del src, dst
    torch.cuda.empty_cache()
    traffic_gbps = 2 * nbytes / 1e6 / ms            # every payload byte is read once and written once
    return {"copy_d2d": {"bound": "hbm", "kernel": "nvs_slab_copy_tma (device-to-device, %d CTAs)" % n_sms,
                         "achieved": traffic_gbps, "peak": peak, "unit": "GB/s", "frac": traffic_gbps / peak,
                         "peak_source": source, "payload_GBps": nbytes / 1e6 / ms, "verified": ok},
            "scan_hash": {"bound": "hbm", "kernel": "nvs_slab_scan (128-bit hash + same-filled test, 4 CTAs/SM)",
                          "achieved": nbytes / 1e6 / scan_ms, "peak": peak, "unit": "GB/s",
                          "frac": nbytes / 1e6 / scan_ms / peak, "peak_source": source, "deterministic": same}}


def probe_main():
    import torch
    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda")
    free_b, total_b = torch.cuda.mem_get_info()
    out = {"hbm_free": free_b, "hbm_total": total_b, "n_gpus_visible": torch.cuda.device_count(),
           "link": measure_link_peak(torch), "peer": measure_peer_peak(torch), "hbm_copy_GBps": measure_hbm_peak(torch)}
    if os.environ.get("NVS_BENCH_PROBE_KERNELS", "1") == "1":
        try:
            out["kernels"] = measure_kernels(torch, *hbm_peak(out))
        except Exception as ex:      # no engine library: report it, the bench itself will fail loudly later
            out["kernels_error"] = repr(ex)
    print("PROBE " + json.dumps(out), flush=True)
    return 0


def run_probes(kernels=True):
    """kernels=False for the reference arm: nothing of ours is loaded anywhere in that arm, probes included."""
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    env["NVS_BENCH_PROBE_KERNELS"] = "1" if kernels else "0"
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--probe"], capture_output=True, text=True, timeout=900, env=env)
    for line in r.stdout.splitlines():
        if line.startswith("PROBE "):
            return json.loads(line[6:])
    raise SystemExit("probe subprocess failed:\n" + r.stdout[-2000:] + r.stderr[-3000:])


def cpu_baseline(sample_gib=4):
    """oracle_slab_move (memcpy restatement of page migration) on one core."""
    lib_path = ROOT / "oracle" / "_ref" / "liboracle.so"
    if not lib_path.exists():
        return {"value": None, "unit": "GB/s", "cores": 1, "kind": "port", "sample": "oracle not built"}
    import numpy as np
    from nvshare_b200.engine import CopyDesc
    lib = C.CDLL(str(lib_path))
    lib.oracle_slab_move.argtypes = [C.c_void_p, C.c_uint32]
    nbytes = sample_gib * GiB
    src = np.ones(nbytes, dtype=np.uint8)
    dst = np.zeros(nbytes, dtype=np.uint8)
    n = nbytes // (2 * MiB)
    arr = (CopyDesc * n)()
    for i in range(n):
        j = (i * 2654435761) % n if n & (n - 1) else (i * 2654435761) & (n - 1)
        arr[i].src, arr[i].dst, arr[i].bytes = src.ctypes.data + j * 2 * MiB, dst.ctypes.data + j * 2 * MiB, 2 * MiB
    lib.oracle_slab_move(arr, n)        # touch
    best = 0.0
    t_all = time.time()
    while time.time() - t_all < 6:
        t0 = time.time()
        lib.oracle_slab_move(arr, n)
        best = max(best, nbytes / 1e9 / (time.time() - t0))
    return {"value": round(best, 2), "unit": "GB/s", "cores": 1, "kind": "port",
            "sample": f"{sample_gib} GiB of 2 MiB slab descriptors, host->host memcpy (oracle_slab_move), best pass in 6 s"}


# ---------------------------------------------------------------- geometry --

def host_memory_budget():
    """Bytes of host RAM this job may still take: the cgroup limit (pinned and UVM
    host pages are charged to it) or MemAvailable."""
    avail = None
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    except OSError:
        pass
    try:
        lim = open("/sys/fs/cgroup/memory.max").read().strip()
        cur = int(open("/sys/fs/cgroup/memory.current").read())
        if lim != "max":
            room = int(lim) - cur
            avail = room if avail is None else min(avail, room)
    except (OSError, ValueError):
        pass
    return avail


def host_memory_needed(impl, clients, footprint, hbm_avail, world=1):
    """What each arm keeps in host RAM: the reference's UVM ends up
    holding every client's pages on the host.  Ours: the shared pool is a budget fixed at creation
    (one HBM's worth, cut to what the cgroup / tmpfs allow: engine.c shp_open) -- what is swapped out
    is the floor it needs; kept copies use whatever else the budget has.  Peer tier: next to nothing."""
    if impl == "reference":
        return clients * footprint * 1.03 + (8 << 30)
    if world > 1:
        return 16 << 30
    swapped = max(clients * footprint - hbm_avail, 0)
    try:   # the scheduler-wide pool lives in /dev/shm; without room there every client pins its own arenas
        vfs = os.statvfs("/dev/shm")
        shared_ok = vfs.f_bavail * vfs.f_frsize >= hbm_avail / 2
    except OSError:
        shared_ok = False
    return (swapped * 1.25 if shared_ok else swapped * clients * 1.15) + (30 << 30)


def pick_fraction(impl, clients, oversub, total_b, forced=0.0, world=1):
    if forced > 0:
        return forced, None
    budget = host_memory_budget()
    frac = 1.0
    while frac > 0.1:
        hbm_avail = total_b * frac
        fp = oversub * hbm_avail / clients
        if budget is None or host_memory_needed(impl, clients, fp, hbm_avail, world) <= budget - (20 << 30):
            break
        frac = round(frac - 0.05, 2)
    note = None
    if frac < 0.999:
        note = (f"host RAM budget {budget / 1e9:.0f} GB cannot hold what the {impl} arm needs at full scale "
                f"({host_memory_needed(impl, clients, oversub * total_b / clients, total_b, world) / 1e9:.0f} GB); "
                f"scaled to {frac:.2f} of the HBM, the rest is held by a ballast process")
    return frac, note


KIND_DEFAULTS = {          # clients, oversubscription, TQ, what the reference script is
    "add": (2, 1.5, 10, "tests/pytorch-add.py"),
    "matmul": (2, 1.5, 30, "tests/tf-matmul.py"),
    "resnet": (2, 1.9, 5, "none (authored: BASELINE config #4)"),
    "llama": (4, 3.0, 5, "none (authored: BASELINE config #5)"),
}


def make_spec(kind, pattern, footprint):
    """Client specification reaching `footprint` bytes of device memory per client."""
    if kind in ("add", "matmul"):
        # live n^2 fp32 blocks -- add: x, y, the result and, while `z = op(x, y)` rebinds, the previous result;
        # matmul: the reference's three (two constants and the product, written in place)
        blocks = 4 if kind == "add" else 3
        n = int(math.floor(math.sqrt(footprint / (4 * blocks))))
        return {"kind": kind, "n": n, "pattern": pattern}, blocks * 4 * n * n
    if kind == "resnet":
        return {"kind": "resnet", "batch": 256, "steps": 4, "tf32": 1, "target_bytes": int(footprint)}, footprint
    # Llama-7B geometry, fp32: 27 GB of weights + a KV cache of batch x context tokens (1 MiB per token)
    ctx = 4096
    batch = max(1, int((footprint - (36 << 30)) // (ctx * (1 << 20))))
    size = "7b" if footprint > (48 << 30) else "small"
    if size == "small":
        batch, ctx = 16, 256
    return {"kind": "llama", "size": size, "batch": batch, "context": ctx, "steps": 8, "tf32": 1,
            "target_bytes": int(footprint)}, footprint


# -------------------------------------------------------------- experiment --

def statistics_mean(xs):
    xs = [x for x in xs if x is not None]
    return sum(xs) / len(xs) if xs else None


def run_experiment(impl, kind, pattern, clients, oversub, tq, warmup, steps, total_b, hbm_fraction, world, out_dir,
                   peer_capacity_frac=0.92, time_limit_s=None, dump=None):
    """One co-located run: calibration (solo, un-hooked), the clients under the chosen library + scheduler,
    analysis.  Returns a dict; never raises for a failed run (reports it)."""
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    hbm_avail = int(total_b * hbm_fraction)
    spec, footprint = make_spec(kind, pattern, oversub * hbm_avail / clients)
    if dump:
        spec["dump"] = str(dump)
    # what MUST come in (and go out) per hand-off: the arriving client's working set minus the share of the
    # HBM the holder does not need -- at best all of that share belongs to the client whose turn is next
    algo_bytes_dir = max(min(footprint, 2 * footprint - hbm_avail), 0.0)
    res = {"kind": kind, "impl": impl, "clients": clients, "tq_s": tq, "steps": steps, "warmup": warmup,
           "hbm_fraction_used": hbm_fraction, "footprint_bytes_per_client": footprint,
           "oversubscription": clients * footprint / hbm_avail, "algorithmic_bytes_per_handoff_per_direction": algo_bytes_dir,
           "spec": {k: v for k, v in spec.items() if k not in ("golden", "dump")}}

    ballast = None
    if hbm_fraction < 0.999:
        ballast_bytes = int(total_b * (1 - hbm_fraction))
        code = ("import torch,time; b=torch.empty(%d,dtype=torch.uint8,device='cuda:0'); torch.cuda.synchronize();"
                "print('BALLAST',flush=True); time.sleep(100000)" % ballast_bytes)
        ballast = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, text=True)
        assert "BALLAST" in ballast.stdout.readline()
    try:
        t0 = time.time()
        try:
            cal = harness.calibrate(spec, out_dir, env=dict(os.environ, CUDA_VISIBLE_DEVICES="0") if world > 1 else None)
        except Exception as ex:
            res.update({"error": f"calibration failed: {ex}", "verified": False})
            return res
        res["calibration"] = {k: v for k, v in cal.items() if k != "golden"}
        res["calibration"]["wall_s"] = time.time() - t0
        if cal.get("golden"):
            spec["golden"] = cal["golden"]
        tau = cal["tau_s"]

        extra = {}
        if world > 1 and impl == "ours":
            extra["NVSHARE_PEERS"] = ",".join(str(i) for i in range(1, world))
            # per peer; empty peer arenas are returned at once, so the clients share the peers' HBM over time
            extra["NVSHARE_PEER_CAPACITY_MIB"] = int(peer_capacity_frac * total_b) >> 20
        # the clients stop as soon as warmup + steps + 2 hand-offs have been seen; this is only the safety limit
        per_handoff = tq + (12 if impl == "ours" else 60) + (0 if kind in ("add",) else 20)
        seconds = (warmup + steps + 3) * per_handoff + 60
        setup_timeout = 1800
        if time_limit_s:             # a sub-run inside somebody else's time limit: never overrun it
            left = time_limit_s - (time.time() - t0)
            # the timed part gets what its hand-offs need first (stall allowance: 4 s for add, 7 s for the models),
            # the clients' setup whatever is left of the limit
            need = (warmup + steps + 2) * (tq + (4 if kind == "add" else 7)) + 10
            setup_timeout = max(45.0, left - need - 20)
            seconds = min(seconds, max(20.0, left - setup_timeout - 20))
        sampler = harness.ClockSampler(out_dir / "clocks.csv")
        sampler.start()
        t0 = time.time()
        try:
            runs = harness.run_clients(impl, out_dir, clients, spec, seconds, tq, extra_env=extra,
                                       stop_after_handoffs=warmup + steps + 2, setup_timeout=setup_timeout)
        except RuntimeError as ex:
            res.update({"error": str(ex), "verified": False})
            return res
        finally:
            res["clocks"] = sampler.stop()
        res["wall_s"] = time.time() - t0
    finally:
        if ballast:
            ballast.kill()
            ballast.wait()

    res["verified"] = all(r["rc"] == 0 and r["meta"].get("summary", {}).get("result") == "PASS" for r in runs)
    res["client_rc"] = [r["rc"] for r in runs]
    timelines = {f"client{i}": r["iters"] for i, r in enumerate(runs)}
    try:
        a = harness.analyse(timelines, warmup, steps, tau=tau)
    except Exception as ex:  # not enough hand-offs: report what happened, loudly
        last_ops = {}
        for i in range(clients):        # what the engines did last: the first thing one wants to know
            f = out_dir / f"engine{i}.jsonl"
            if f.exists():
                last_ops[f"client{i}"] = [l[:400] for l in f.read_text().splitlines() if '"op":"pin"' not in l][-6:]
        res.update({"error": str(ex), "verified": False, "engine_last_ops": last_ops,
                    "stderr_tails": {f"client{i}": r["err_tail"][-800:] for i, r in enumerate(runs)},
                    "host_memory_budget": host_memory_budget()})
        return res
    stall = a["stall_per_handoff_s"]
    res["analysis"] = a
    res["stall_ms_per_handoff"] = 1e3 * stall
    res["iter_per_s"] = a["iter_per_s"]
    res["e2e_GBps"] = (2 * algo_bytes_dir / 1e9) / stall if stall > 0 else None
    if not res["verified"]:
        res["stderr_tails"] = {f"client{i}": r["err_tail"][-800:] for i, r in enumerate(runs)}

    if impl == "ours":
        paths = [out_dir / f"engine{i}.jsonl" for i in range(clients)]
        recs = harness.engine_records(paths, a["t_start"], a["t_end"])
        ev = [r for r in recs if r["op"] == "evict"]
        fe = [r for r in recs if r["op"] == "fetch" and (r["bytes"] or r.get("elided_bytes"))]

        def rate(rs, key="bytes", ms="copy_ms"):
            t = sum(r[ms] for r in rs)
            return sum(r[key] for r in rs) / 1e6 / t if t > 0 else None
        res["device"] = {
            "evict_GBps": rate(ev), "fetch_GBps": rate(fe), "scan_GBps": rate(ev, "scanned_bytes", "scan_ms"),
            "bytes_evicted": sum(r["bytes"] for r in ev), "bytes_fetched": sum(r["bytes"] for r in fe),
            "bytes_skipped_clean": sum(r.get("clean_bytes", 0) for r in ev),
            "bytes_elided_same_filled": sum(r.get("elided_bytes", 0) for r in ev),
            "bytes_scanned": sum(r.get("scanned_bytes", 0) for r in ev),
            "host_bytes": {"out": sum(r["host_bytes"] for r in ev), "in": sum(r["host_bytes"] for r in fe)},
            "peer_bytes": {"out": sum(r["peer_bytes"] for r in ev), "in": sum(r["peer_bytes"] for r in fe)},
            "copy_ms": {"evict": sum(r["copy_ms"] for r in ev), "fetch": sum(r["copy_ms"] for r in fe)},
            "scan_ms": sum(r.get("scan_ms", 0) for r in ev), "scan_launches": sum(r.get("scan_launches", 0) for r in ev),
            "copy_kernel_launches": sum(r["launches"] - r.get("scan_launches", 0) for r in ev) + sum(1 for r in fe if r["peer_bytes"] and r["launches"]),
            "kernel_launches": sum(r["launches"] for r in ev + fe), "ce_calls": sum(r.get("ce_calls", 0) for r in ev + fe),
            "evicts": len(ev), "fetches": len(fe),
            "map_ms_mean": statistics_mean([r["map_ms"] for r in ev + fe]),
            "wait_ms_mean": statistics_mean([r["wait_ms"] for r in fe]),
            "wall_ms_mean": {"evict": statistics_mean([r["wall_ms"] for r in ev]),
                             "fetch": statistics_mean([r["wall_ms"] for r in fe])},
            "retained_bytes_last": max([r.get("retained_bytes", 0) for r in recs] or [0]),
            "pool_used_max": max([r.get("pool_used", 0) for r in recs] or [0]),
        }
        if algo_bytes_dir > 0 and fe and ev:
            # per transfer that completed inside the window (the window may hold one more of them than timed steps)
            res["device"]["link_bytes_over_algorithmic"] = {
                "in": res["device"]["bytes_fetched"] / len(fe) / algo_bytes_dir,
                "out": res["device"]["bytes_evicted"] / len(ev) / algo_bytes_dir}
        led = [r for r in recs if "gl_lent" in r]
        if led:         # peer tier: the cross-process GPU ledger as the engines saw it at their transfers (gpu_ledger.c)
            res["device"]["gpu_ledger"] = {
                "tracked_peers": max(r["gl_tracked_peers"] for r in led),
                "lent_bytes_max": max(r["gl_lent"] for r in led),              # all clients' arenas on the peers, per the ledger
                "one_client_lent_bytes_max": max(r["gl_my_lent"] for r in led),
                "one_client_arena_bytes_max": max(r["peer_pool_bytes"] for r in led),   # what that engine itself holds mapped
                "own_claim_matches_arenas": all(r["gl_my_lent"] == r["peer_pool_bytes"] for r in led if r["gl_tracked_peers"]),
                "refusals": max(r["gl_refusals"] for r in led)}
        pins = [r for r in harness.engine_records(paths, 0, 1e18) if r["op"] == "pin"]
        if pins:        # where the pinned pool's pages ended up (engine.c numa_init): the last report covers the whole pool
            last = max(pins, key=lambda r: r["t"])
            res["device"]["pool_pages_per_numa_node"] = last["pages_per_node"]
    return res


def roofline_objects(exp, probe, world):
    """The `roofline` family of keys from one experiment of our arm."""
    d = exp.get("device") or {}
    link = probe["link"]
    out = {}
    scan_launches = max(d.get("evicts", 0), 1)
    hbm_pk, hbm_src = hbm_peak(probe)
    scan = {"bound": "hbm", "kernel": "nvs_slab_scan", "achieved": d.get("scan_GBps"), "peak": hbm_pk, "unit": "GB/s",
            "frac": d["scan_GBps"] / hbm_pk if d.get("scan_GBps") else None, "peak_source": hbm_src,
            "algorithmic_bytes_total": d.get("bytes_scanned"),
            "note": "bytes the scan/hash launches of the timed evictions read / their CUDA-event time; alone on an idle GPU: "
                    "see roofline_kernels.scan_hash.  The peak is the measured COPY figure (read + write traffic of b.copy_(a)); "
                    "a read-only pass has no write turn-arounds and can exceed it (frac > 1)"}
    scan["algorithmic_bytes_per_launch"] = d["bytes_scanned"] / d["scan_launches"] if d.get("scan_launches") else None
    scan["launches"] = d.get("scan_launches")
    if world == 1:
        out["roofline"] = scan
        out["roofline_link"] = {
            "bound": "pcie", "engine": "copy engines (cuMemcpyAsync), both directions",
            "evict": {"achieved": d.get("evict_GBps"), "peak": link["d2h"],
                      "frac": d["evict_GBps"] / link["d2h"] if d.get("evict_GBps") else None},
            "fetch": {"achieved": d.get("fetch_GBps"), "peak": link["h2d"],
                      "frac": d["fetch_GBps"] / link["h2d"] if d.get("fetch_GBps") else None},
            "unit": "GB/s", "peak_source": "cuMemcpyAsync pinned<->HBM measured in this run, one direction at a time "
                                           "(nominal PCIe Gen5 x16: 63.0 GB/s)"}
    else:
        peer = probe.get("peer") or {}
        pk_out, pk_in = peer.get("out"), peer.get("in")
        per_dir = [g for g in (d.get("evict_GBps"), d.get("fetch_GBps")) if g]
        achieved = sum(per_dir) / len(per_dir) if per_dir else None
        pk = (pk_out + pk_in) / 2 if pk_out and pk_in else None
        out["roofline"] = {"bound": "nvlink", "kernel": "nvs_slab_copy_tma", "achieved": achieved, "peak": pk, "unit": "GB/s",
                           "frac": achieved / pk if achieved and pk else None,
                           "evict": {"achieved": d.get("evict_GBps"), "peak": pk_out,
                                     "frac": d["evict_GBps"] / pk_out if d.get("evict_GBps") and pk_out else None},
                           "fetch": {"achieved": d.get("fetch_GBps"), "peak": pk_in,
                                     "frac": d["fetch_GBps"] / pk_in if d.get("fetch_GBps") and pk_in else None},
                           "peak_source": "cuMemcpyPeer GPU0<->GPU1 measured in this run" if pk_out else "not measured",
                           "algorithmic_bytes_per_launch": ((d["peer_bytes"]["out"] + d["peer_bytes"]["in"]) / d["copy_kernel_launches"]
                                                            if d.get("copy_kernel_launches") else None)}
        out["roofline_scan"] = scan
    out["roofline_kernels"] = probe.get("kernels")
    return out


def main():
    args = parse_args()
    if args.probe:
        return probe_main()
    rank, world, local = dist_env()
    clients_d, oversub_d, tq_d, _ = KIND_DEFAULTS[args.kind]
    args.clients = args.clients or clients_d
    args.oversub = args.oversub or oversub_d
    args.tq = args.tq or tq_d

    # reference arm: rank 0 alone runs and prints; the other ranks exit 0 without work
    if args.impl == "reference" and rank != 0:
        return 0
    use_dist = world > 1 and args.impl != "reference"
    if use_dist:
        import torch
        import torch.distributed as dist
        import datetime
        if torch.cuda.is_available():
            torch.cuda.set_device(local)
        dist.init_process_group("nccl" if torch.cuda.is_available() else "gloo", rank=rank, world_size=world,
                                timeout=datetime.timedelta(minutes=60))
        # create the communicator now, while GPU 0 is still empty; the data-path work then runs on rank 0
        # alone (the path shards by slab over the peers' HBM, not by rank) and everybody meets again below
        dist.barrier()

    result = None
    t_region = 0.0
    if rank == 0:
        result, t_region = run_rank0(args, world)
    if use_dist:
        dist.barrier()
        t = torch.tensor([t_region], dtype=torch.float64, device="cuda" if torch.cuda.is_available() else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)       # max over ranks (only rank 0 does data-path work)
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(result), flush=True)
        return 0 if result.get("verified", True) else 1
    return 0


def run_rank0(args, world):
    paths = harness.impl_paths(args.impl)
    if not paths["lib"].exists():
        if args.impl == "reference":
            return {"impl": "reference", "unavailable": "oracle/_ref not built (reference sources absent at build time)"}, 0.0
        raise SystemExit("nvshare_b200/_build is missing: run __graft_entry__.build() first")
    if args.impl == "reference" and args.kind in ("resnet", "llama"):
        return {"impl": "reference", "unavailable": "the model configurations are authored by this repository; "
                "the reference arm runs the reference's own two workloads (add, matmul)"}, 0.0

    ncpu = os.cpu_count()
    probe = run_probes(kernels=args.impl == "ours")
    total_b = probe["hbm_total"]
    cpu = cpu_baseline() if (args.impl == "ours" and world == 1) or args.impl == "reference" else None

    frac, scale_note = pick_fraction(args.impl, args.clients, args.oversub, total_b, args.hbm_fraction, world)
    out_dir = Path(args.keep) if args.keep else Path(tempfile.mkdtemp(prefix="nvs_bench_"))
    t0 = time.time()
    exp = run_experiment(args.impl, args.kind, args.pattern, args.clients, args.oversub, args.tq, args.warmup, args.steps,
                         total_b, frac, world if args.impl == "ours" else 1, out_dir / "main",
                         dump=Path(args.dump_outputs).resolve() if getattr(args, "dump_outputs", "") else None)
    _, _, _, ref_script = KIND_DEFAULTS[args.kind]
    sp = exp["spec"]
    what = (f"fp32 [n,n] n={sp['n']} ({args.pattern})" if "n" in sp else
            f"batch {sp.get('batch')}" + (f", context {sp.get('context')}, {sp.get('size')}" if args.kind == "llama" else ""))
    line = {
        "metric": METRIC, "unit": "GB/s", "impl": args.impl, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "verified": bool(exp.get("verified")),
        "config": {
            "workload": f"{args.clients}x {args.kind} {what}, restated {ref_script}, footprint "
                        f"{exp['footprint_bytes_per_client'] / 1e9:.1f} GB/client = {exp['oversubscription']:.2f}x of "
                        f"{total_b * frac / 1e9:.1f} GB HBM",
            "clients": args.clients, "oversubscription": exp["oversubscription"], "tq_s": args.tq,
            "tq_note": "BASELINE.md names TQ 30 and 5; 10 s keeps K=20 hand-offs of BOTH arms inside the driver's time "
                       "limit and is the smallest TQ the reference's README allows (\"don't set TQ < 10\")",
            "hbm_bytes": total_b, "hbm_fraction_used": frac, "scale_note": scale_note,
            "backing_tier": "peer-HBM over NVLink (GPUs 1..%d) + pinned host" % (world - 1) if world > 1 and args.impl == "ours"
                            else "pinned host DRAM over PCIe Gen5 x16",
            "l2_policy": "inputs (>= tens of GB per hand-off) exceed the 50 MB L2",
            "algorithmic_bytes_per_handoff_per_direction": exp["algorithmic_bytes_per_handoff_per_direction"],
            "host_cores": ncpu,
        },
        "link_peak_GBps_measured": probe["link"], "peer_peak_GBps_measured": probe.get("peer"),
    }
    if "error" in exp:
        line.update({"error": exp["error"], "verified": False, "diagnostics": {k: exp.get(k) for k in
                     ("client_rc", "stderr_tails", "engine_last_ops", "host_memory_budget", "calibration")}})
        line["wall_s_total"] = time.time() - t0
        return line, line["wall_s_total"]
    a = exp["analysis"]
    line.update({
        "ms_per_step": 1e3 * a["window_s"] / args.steps, "iter_per_s": a["iter_per_s"],
        "iter_per_s_resident": a["iter_per_s_resident"], "tau_s": exp["calibration"]["tau_s"], "tau_source": a["tau_source"],
        "tau_own_p10_s": a["tau_own_p10_s"], "stall_ms_per_handoff": exp["stall_ms_per_handoff"],
        "first_iter_gap_ms": [1e3 * g for g in a["first_iter_gap_s"]], "gpu_busy_frac": a["gpu_busy_frac"],
        "clocks": exp["clocks"],
    })
    if "analysis_error" in a:
        line["analysis_error"] = a["analysis_error"]
    if exp.get("stderr_tails"):
        line["stderr_tails"] = exp["stderr_tails"]
    e2e = exp["e2e_GBps"]

    if args.impl == "ours":
        d = exp["device"]
        moved = d["bytes_evicted"] + d["bytes_fetched"]
        dev_ms = d["copy_ms"]["evict"] + d["copy_ms"]["fetch"]
        line["value"] = moved / 1e6 / dev_ms if dev_ms else None
        line["gpu_launches"] = d["kernel_launches"]
        line["ce_calls"] = d["ce_calls"]
        line["device"] = d
        line.update(roofline_objects(exp, probe, world))
        line["e2e"] = {"value": e2e, "unit": "GB/s", "iter_per_s": a["iter_per_s"],
                       "h2d_bytes_per_step": (d["host_bytes"]["in"] + d["peer_bytes"]["in"]) / max(args.steps, 1),
                       "d2h_bytes_per_step": (d["host_bytes"]["out"] + d["peer_bytes"]["out"]) / max(args.steps, 1),
                       "definition": "2 x algorithmic bytes per hand-off / stall per hand-off seen by the application; "
                                     "the per-step bytes are what really crossed the link (unchanged slabs are not copied again)"}
        if cpu:
            line["cpu_baseline"] = cpu
        if not args.no_extras:
            extras(args, line, probe, world, total_b, frac, out_dir, T_START)
            config1(args, line, world, out_dir)
    else:
        line["value"] = e2e
        line["gpu_launches"] = 0
        line["e2e"] = {"value": e2e, "unit": "GB/s", "iter_per_s": a["iter_per_s"], "h2d_bytes_per_step": 0,
                       "d2h_bytes_per_step": 0}
        line["cpu_baseline"] = {"value": e2e, "unit": "GB/s", "cores": ncpu, "kind": "reference",
                                "sample": "the reference has no CPU compute path: this is its UVM page-fault path "
                                          "(cuMemAllocManaged) on the same box, same workload; host cores only service faults"}
        if not args.no_extras:
            config1(args, line, world, out_dir)
    line["wall_s_total"] = time.time() - t0
    if not args.keep:
        shutil.rmtree(out_dir, ignore_errors=True)
    return line, line["wall_s_total"]


def brief(exp):
    """A sub-run, cut down to what a reader of the JSON line needs."""
    keep = ("kind", "impl", "clients", "tq_s", "steps", "warmup", "hbm_fraction_used", "footprint_bytes_per_client",
            "oversubscription", "algorithmic_bytes_per_handoff_per_direction", "verified", "stall_ms_per_handoff", "iter_per_s",
            "e2e_GBps", "error", "wall_s", "client_rc", "stderr_tails", "engine_last_ops", "spec")
    out = {k: exp[k] for k in keep if k in exp}
    if "analysis" in exp:
        a = exp["analysis"]
        out.update({"tau_s": exp["calibration"]["tau_s"], "iter_per_s_resident": 1.0 / exp["calibration"]["tau_s"],
                    "first_iter_gap_ms": [1e3 * g for g in a["first_iter_gap_s"]], "window_s": a["window_s"]})
        if "analysis_error" in a:
            out["analysis_error"] = a["analysis_error"]
    if "device" in exp:
        d = exp["device"]
        out["device"] = {k: d[k] for k in ("evict_GBps", "fetch_GBps", "bytes_evicted", "bytes_fetched", "bytes_skipped_clean",
                                           "bytes_elided_same_filled", "peer_bytes", "host_bytes", "kernel_launches", "ce_calls",
                                           "map_ms_mean", "wait_ms_mean", "wall_ms_mean", "gpu_ledger") if k in d}
    return out


# A `bench.py --gpus N` run has to finish inside 10 minutes; the sub-runs only get what the headline has left
# of a budget well inside that, and say so when they had to be skipped or cut.
TOTAL_BUDGET_S = 480.0


def extras(args, line, probe, world, total_b, frac, out_dir, t_bench_start):
    """Sub-runs that make the other BASELINE configurations and a same-configuration pair driver-visible.
    Each is independent: a failure is reported inside its own record and never costs the headline."""
    if args.kind != "add":
        return

    def left():
        return TOTAL_BUDGET_S - (time.time() - t_bench_start)
    if world == 1:
        ref_frac, _ = pick_fraction("reference", args.clients, args.oversub, total_b, 0.0, 1)
        if ref_frac < frac - 0.01 and left() < 240:
            line["same_scale"] = {"skipped": f"only {left():.0f} s of the run's time budget left"}
        elif ref_frac < frac - 0.01:
            try:
                # (five hand-offs of warm-up like the headline: each client has to evict twice before the
                # engine knows which of its chunks are worth keeping copies of)
                exp = run_experiment("ours", "add", args.pattern, args.clients, args.oversub, args.tq, min(max(args.warmup, 5), 6),
                                     min(args.steps, 4), total_b, ref_frac, 1, out_dir / "same_scale", time_limit_s=left())
                line["same_scale"] = brief(exp)
                line["same_scale"]["why"] = ("the reference arm cannot hold 2 x footprint in this box's host RAM and runs at "
                                             "this fraction of the HBM; this is our arm in that very configuration")
            except Exception as ex:
                line["same_scale"] = {"error": repr(ex)}
    line["configs"] = {}
    plan = []
    if world == 2:
        plan.append(("config4_resnet50_train_x2_2xHBM_peer_tier", "resnet"))
    if world == 8:
        plan.append(("config5_llama7b_decode_x4_3xHBM_peer_tier", "llama"))
    for name, kind in plan:
        clients, oversub, tq, _ = KIND_DEFAULTS[kind]
        if left() < 240:
            line["configs"][name] = {"skipped": f"only {left():.0f} s of the run's time budget left", "verified": None}
            continue
        try:
            exp = run_experiment("ours", kind, "pos", clients, oversub, tq, 2, 4, total_b, 1.0, world, out_dir / name,
                                 peer_capacity_frac=0.97, time_limit_s=left())
            line["configs"][name] = brief(exp)
        except Exception as ex:
            line["configs"][name] = {"error": repr(ex), "verified": False}


def config1(args, line, world, out_dir):
    """BASELINE config #1, the reference's own CPU-runnable case: this arm's daemon under scripted clients
    (harness.scheduler_pingpong; a few seconds, no GPU).  Both arms carry it, so that the pair is in the
    driver's record; N = 1 only, where nothing else competes for the host cores."""
    if world != 1 or args.kind != "add":
        return
    if time.time() - T_START > TOTAL_BUDGET_S - 60:
        line.setdefault("configs", {})["config1_scheduler_cpu_2_clients"] = {"skipped": "the run's time budget is spent"}
        return
    try:
        rec = harness.scheduler_pingpong(args.impl, out_dir / "config1", clients=2, cycles=20000, trials=5)
    except Exception as ex:
        rec = {"error": repr(ex)}
    line.setdefault("configs", {})["config1_scheduler_cpu_2_clients"] = rec


if __name__ == "__main__":
    sys.exit(main())
