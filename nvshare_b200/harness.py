"""Measurement harness for BASELINE configs #2/#3: N co-located clients of
nvshare_b200/workloads.py under a libnvshare.so + nvshare-scheduler pair (ours
or the reference's), and the analysis that turns their per-iteration logs into
the headline numbers.  Used by bench.py for BOTH arms, so the two are measured
by identical code.

Definitions (SURVEY 8d / BASELINE.md section 2):
  hand-off     a change of the client that is completing iterations
  tau          steady iteration time of a client with its working set resident
               (10th percentile of its iteration durations)
  lost time    window wall time minus (iterations completed in the window) x tau,
               summed over the clients; divided by the number of hand-offs in the
               window it is the stall per hand-off.  Slow post-resume iterations
               (the reference's fault storm) count in full.
  algorithmic bytes per hand-off
               what MUST cross the link so that the next client is resident:
               (n_clients * F - C_avail) in, the same amount out, where F is a
               client's footprint and C_avail the HBM the clients share
  e2e swap GB/s = algorithmic bytes per hand-off / stall per hand-off
"""
from __future__ import annotations

import json
import os
import shutil
import signal
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
BUILD = ROOT / "nvshare_b200" / "_build"
REF = ROOT / "oracle" / "_ref"


def impl_paths(impl: str):
    base = BUILD if impl == "ours" else REF
    return {"lib": base / "libnvshare.so", "sched": base / "nvshare-scheduler", "ctl": base / "nvsharectl"}


def preload_for(impl, lib):
    """LD_PRELOAD for a process of `impl`: the reference's binaries only know /var/run/nvshare, which an ordinary
    user cannot create; oracle/_ref/libsockdir.so, in front of them, takes NVSHARE_SOCK_DIR instead."""
    first = [] if impl == "ours" else [str(REF / "libsockdir.so")]
    rest = [os.environ["LD_PRELOAD"]] if os.environ.get("LD_PRELOAD") else []
    return ":".join(first + [str(lib)] + rest) if lib else ":".join(first + rest)


# ----------------------------------------------------------------- analysis --

def load_iters(path):
    """[(t_complete, index)] for one client, plus its setup/summary records."""
    iters, meta = [], {}
    for line in Path(path).read_text().splitlines():
        try:
            r = json.loads(line)
        except json.JSONDecodeError:
            continue
        if r.get("event") == "iter":
            iters.append(r["t"])
        elif r.get("event") in ("setup_done", "summary"):
            meta[r["event"]] = r
    return iters, meta


def steady_tau(ts):
    """10th percentile of a client's own iteration durations.  Only a cross-check: when a client
    never reaches resident speed inside its quantum (the reference at full scale keeps faulting)
    this over-estimates the resident iteration time and hides lost time -- the analysis uses the
    solo calibration (calibrate()) instead."""
    d = sorted(b - a for a, b in zip(ts, ts[1:]) if b > a)
    if not d:
        return float("nan")
    return d[max(0, len(d) // 10)]


def merged_timeline(clients):
    """clients: {name: [t...]} -> sorted [(t, name)]"""
    ev = [(t, n) for n, ts in clients.items() for t in ts]
    ev.sort()
    return ev


def handoff_boundaries(timeline):
    """Times at which the completing client changes: (t_last_of_previous, prev, nxt)."""
    out = []
    for (t0, a), (t1, b) in zip(timeline, timeline[1:]):
        if a != b:
            out.append((t0, a, b))
    return out


def analyse(clients, warmup, steps, tau=None):
    """clients: {name: [iteration completion times]}.  Returns the window metrics
    over exactly `steps` hand-offs after `warmup` hand-offs, or raises.

    tau: resident iteration time of this workload from a solo, un-hooked, un-oversubscribed
    calibration run (seconds).  Without it the clients' own 10th percentile is used and the
    result is marked as such."""
    tl = merged_timeline(clients)
    bounds = handoff_boundaries(tl)
    if len(bounds) < warmup + steps + 1:
        raise RuntimeError(f"only {len(bounds)} hand-offs observed, need {warmup + steps + 1}")
    t_start = bounds[warmup][0]
    t_end = bounds[warmup + steps][0]
    own = {n: steady_tau(ts) for n, ts in clients.items()}
    taus = {n: (tau if tau else own[n]) for n in clients}
    n_iters = {n: sum(1 for t in ts if t_start < t <= t_end) for n, ts in clients.items()}
    busy = sum(n_iters[n] * taus[n] for n in clients)
    wall = t_end - t_start
    lost = wall - busy                       # NOT clamped: a negative value means the analysis does not apply
    # per-hand-off gap: last iteration of the leaving client -> first iteration of the arriving one
    gaps = []
    for k in range(warmup, warmup + steps):
        t_last, a, b = bounds[k]
        t_first = next(t for t, n in tl if t > t_last and n == b)
        gaps.append(t_first - t_last - taus[b])
    errors = []
    if lost < 0:
        errors.append(f"lost time {lost:.3f} s < 0: the clients completed more iterations than fit the window at tau")
    if any(g < -0.5 * min(taus.values()) for g in gaps):
        errors.append("negative first-iteration gap: iterations of two clients overlap, hand-offs are not clean")
    out = {
        "window_s": wall, "t_start": t_start, "t_end": t_end, "handoffs": steps,
        "iters": n_iters, "tau_s": taus, "tau_source": "solo un-hooked calibration" if tau else "own 10th percentile",
        "tau_own_p10_s": own, "iter_per_s": sum(n_iters.values()) / wall,
        "iter_per_s_resident": {n: 1.0 / taus[n] for n in clients},
        "lost_s": lost, "stall_per_handoff_s": lost / steps, "first_iter_gap_s": gaps,
        "gpu_busy_frac": busy / wall,
    }
    if errors:
        out["analysis_error"] = errors
    return out


def engine_records(paths, t_start, t_end):
    """Engine stats lines (ours only) whose operation ended inside the window."""
    recs = []
    for p in paths:
        p = Path(p)
        if not p.exists():
            continue
        for line in p.read_text().splitlines():
            try:
                r = json.loads(line)
            except json.JSONDecodeError:
                continue
            if t_start < r.get("t", 0) <= t_end + 1.0:
                recs.append(r)
    return recs


# ------------------------------------------------------------------ running --

class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region.  Once a second:
    every sample is a round of NVML queries that take driver locks the hand-off's cuMemUnmap /
    cuMemCreate calls also need."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, path, gpu=0):
        self.path = Path(path)
        self.p = None
        self.gpu = gpu

    def start(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), f"--query-gpu={self.Q}",
                                       "--format=csv,noheader,nounits", "-lms", "1000"],
                                      stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except FileNotFoundError:
            self.p = None

    def stop(self, t_start=None, t_end=None):
        if self.p:
            self.p.terminate()
            try:
                self.p.wait(timeout=5)
            except subprocess.TimeoutExpired:
                self.p.kill()
        sm, smax, reasons = [], [], set()
        if self.path.exists():
            for line in self.path.read_text().splitlines():
                f = [x.strip() for x in line.split(",")]
                if len(f) < 9:
                    continue
                try:
                    sm.append(float(f[1])); smax.append(float(f[2]))
                except ValueError:
                    continue
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(smax), "reasons": sorted(reasons), "samples": len(sm)}


def start_scheduler(impl, sock_dir, log_path, tq, debug=True, cpus=None):
    paths = impl_paths(impl)
    env = dict(os.environ)
    if debug:
        env["NVSHARE_DEBUG"] = "1"
    else:
        env.pop("NVSHARE_DEBUG", None)
    env["NVSHARE_SOCK_DIR"] = str(sock_dir)
    if impl != "ours":
        env["LD_PRELOAD"] = preload_for(impl, None)
    sock = Path(sock_dir) / "scheduler.sock"
    if sock.exists():
        sock.unlink()
    log = open(log_path, "wb")
    p = subprocess.Popen([str(paths["sched"])], env=env, stdout=log, stderr=subprocess.STDOUT,
                         preexec_fn=(lambda: os.sched_setaffinity(0, cpus)) if cpus else None)
    deadline = time.time() + 10
    while not sock.exists():
        if p.poll() is not None or time.time() > deadline:
            raise RuntimeError(f"{impl} nvshare-scheduler did not start; see {log_path}")
        time.sleep(0.02)
    time.sleep(0.1)
    r = subprocess.run([str(paths["ctl"]), "-T", str(int(tq))], env=env, capture_output=True, text=True)
    if r.returncode != 0:
        p.kill()
        raise RuntimeError(f"nvsharectl -T failed: {r.stderr}")
    return p


def sock_dir_for(out_dir):
    """Where the daemon listens: out_dir/sock unless the socket's path would not fit a Unix socket address
    (107 bytes), then a fresh directory under /tmp."""
    d = Path(out_dir) / "sock"
    return d if len(str(d / "scheduler.sock")) <= 107 else Path(tempfile.mkdtemp(prefix="nvs-sock-", dir="/tmp"))


def scheduler_pingpong(impl, out_dir, clients=2, cycles=20000, trials=5):
    """BASELINE config #1 (CPU only): the daemon of `impl` and `clients` scripted clients that do nothing but
    REQ_LOCK -> LOCK_OK -> LOCK_RELEASED (tools/pingpong.c, the same binary against both daemons).  No GPU, no
    library of ours or of the reference in the clients: what is timed is the daemon's hand-off path.

    Where the kernel puts three mostly-sleeping threads decides the result more than the daemon does (a wake-up
    across cores costs ~20 us on a virtual machine, a context switch on one core ~2 us: the same daemon does
    20 k or 85 k hand-offs/s depending on it), so the placement is fixed and both are measured:
      same_core       daemon and clients on one core     -> the daemon's own path length
      separate_cores  daemon on one core, clients on two -> wake-up latency dominated
    Several trials per placement against one daemon; the median trial is the record, all of them are listed."""
    from .build import ORACLE_OUT
    tool = ORACLE_OUT / "pingpong"
    if not tool.exists():
        raise RuntimeError(f"{tool} is missing: run __graft_entry__.build()")
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    sock_dir = sock_dir_for(out_dir)
    sock_dir.mkdir(parents=True, exist_ok=True)
    env = dict(os.environ)
    env.pop("LD_PRELOAD", None)
    cpus = sorted(os.sched_getaffinity(0))
    placements = {"same_core": ({cpus[-1]}, {cpus[-1]})}
    if len(cpus) >= 3:
        placements["separate_cores"] = ({cpus[-1]}, set(cpus[-3:-1]))
    out = {"impl": impl, "clients": clients, "cycles_per_client": cycles, "trials": trials, "host_cores": os.cpu_count(),
           "what": "REQ_LOCK -> LOCK_OK -> LOCK_RELEASED cycles of scripted clients against this arm's nvshare-scheduler "
                   "over the Unix socket (537-byte frames), CPU only; per placement the median of the trials"}
    for name, (sched_cpus, client_cpus) in placements.items():
        sched = start_scheduler(impl, sock_dir, out_dir / f"scheduler_{name}.log", 30, debug=False, cpus=sched_cpus)
        runs = []
        try:
            for _ in range(trials):
                r = subprocess.run([str(tool), str(sock_dir / "scheduler.sock"), str(clients), str(cycles)], env=env,
                                   capture_output=True, text=True, timeout=120,
                                   preexec_fn=lambda c=client_cpus: os.sched_setaffinity(0, c))
                if r.returncode != 0:
                    raise RuntimeError(f"pingpong against the {impl} daemon failed: {r.stderr[-500:]}")
                runs.append(json.loads(r.stdout.strip().splitlines()[-1]))
        finally:
            stop_process(sched)
            if sock_dir.parent != out_dir:
                shutil.rmtree(sock_dir, ignore_errors=True)
        runs.sort(key=lambda x: x["handoffs_per_s"])
        med = runs[len(runs) // 2]
        out[name] = {"handoffs_per_s": med["handoffs_per_s"], "req_to_lock_ok_us": med["req_to_lock_ok_us"],
                     "handoffs_per_s_all_trials": [x["handoffs_per_s"] for x in runs],
                     "daemon_cpus": sorted(sched_cpus), "client_cpus": sorted(client_cpus)}
    out["handoffs_per_s"] = out["same_core"]["handoffs_per_s"]
    return out


def stop_process(p, timeout=10):
    if p is None or p.poll() is not None:
        return
    p.send_signal(signal.SIGTERM)
    try:
        p.wait(timeout=timeout)
    except subprocess.TimeoutExpired:
        p.kill()
        p.wait()


def count_handoffs(out_dir, n_clients):
    clients = {}
    for i in range(n_clients):
        f = Path(out_dir) / f"client{i}.jsonl"
        clients[f"client{i}"] = load_iters(f)[0] if f.exists() else []
    return len(handoff_boundaries(merged_timeline(clients)))


def client_cmd(spec, log, tag, barrier="", stop_file="", seconds=0.0, extra=()):
    """Command line of one client.  spec: {"kind": add|matmul, "n":, "pattern":} or
    {"kind": resnet|llama, "steps":, "batch":, ...}."""
    if spec["kind"] in ("add", "matmul"):
        cmd = [sys.executable, "-m", "nvshare_b200.workloads", "--kind", spec["kind"], "--n", str(spec["n"]),
               "--iters", str(spec.get("iters", 100000000)), "--pattern", spec["pattern"]]
        if spec.get("dump"):
            cmd += ["--dump-outputs", str(spec["dump"])]
    else:
        cmd = [sys.executable, "-m", "nvshare_b200.workloads_models", "--kind", spec["kind"],
               "--steps", str(spec.get("steps", 6)), "--batch", str(spec.get("batch", 16)), "--tf32", str(spec.get("tf32", 0))]
        if spec["kind"] == "llama":
            cmd += ["--size", spec.get("size", "small"), "--context", str(spec.get("context", 32))]
        if spec.get("target_bytes"):
            cmd += ["--target-bytes", str(int(spec["target_bytes"]))]
        if spec.get("golden"):
            cmd += ["--golden", str(spec["golden"])]
    cmd += ["--seconds", str(seconds), "--log", str(log), "--tag", tag]
    if barrier:
        cmd += ["--start-barrier", str(barrier)]
    if stop_file:
        cmd += ["--stop-file", str(stop_file)]
    return cmd + list(extra)


def calibrate(spec, out_dir, env=None, timeout=1800):
    """Solo, un-hooked, un-oversubscribed run of the same application: its resident iteration
    time tau (median, first iterations dropped) and -- for the model workloads -- the golden
    numbers every hooked round is compared with.  No LD_PRELOAD, no scheduler."""
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    log = out_dir / "calibration.jsonl"
    env = dict(env or os.environ, PYTHONPATH=str(ROOT) + (":" + os.environ["PYTHONPATH"] if os.environ.get("PYTHONPATH") else ""))
    env.pop("LD_PRELOAD", None)
    if spec["kind"] in ("add", "matmul"):
        cal = dict(spec, pattern="ones", iters=spec.get("calibration_iters", 6 if spec["kind"] == "matmul" else 40), dump=None)
        cmd = client_cmd(cal, log, "calibration", extra=["--no-verify"])
        golden = None
    else:
        golden = out_dir / "golden.json"
        cal = dict(spec, golden=None, target_bytes=0)
        cmd = client_cmd(cal, log, "calibration", extra=["--rounds", "3", "--write-golden", str(golden)])
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    if r.returncode != 0:
        raise RuntimeError(f"calibration run failed: {r.stderr[-2000:]}")
    ts, meta = load_iters(log)
    skip = 4 if spec["kind"] == "add" else (1 if spec["kind"] == "matmul" else int(spec.get("steps", 6)))
    d = sorted(b - a for a, b in zip(ts[skip:], ts[skip + 1:]) if b > a)
    if not d:
        raise RuntimeError("calibration run produced no iterations")
    return {"tau_s": d[len(d) // 2], "tau_min_s": d[0], "iters": len(ts), "golden": str(golden) if golden else None,
            "setup_s": meta.get("setup_done", {}).get("setup_s"), "torch_reserved": meta.get("setup_done", {}).get("torch_reserved")}


def run_clients(impl, out_dir, n_clients, spec, seconds, tq, extra_env=None, start_stagger=0.0,
                stop_after_handoffs=0, gpu=None, setup_timeout=1800):
    """Run the co-located clients until `stop_after_handoffs` hand-offs have been
    observed (or `seconds` elapsed); each client then verifies its results.
    Returns per-client dicts."""
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    paths = impl_paths(impl)
    sock_dir = sock_dir_for(out_dir)
    sock_dir.mkdir(parents=True, exist_ok=True)
    sched = start_scheduler(impl, sock_dir, out_dir / "scheduler.log", tq)
    barrier = out_dir / "go"
    stop_file = out_dir / "stop"
    for f in (barrier, stop_file):
        if f.exists():
            f.unlink()
    procs = []
    try:
        for i in range(n_clients):
            # keep whatever is already preloaded (e.g. a profiler's injection library) behind ours, and
            # whatever is on PYTHONPATH (the driver's sitecustomize hook records which .so files we load)
            preload = preload_for(impl, paths["lib"])
            pypath = str(ROOT) + (":" + os.environ["PYTHONPATH"] if os.environ.get("PYTHONPATH") else "")
            env = dict(os.environ, LD_PRELOAD=preload, PYTHONPATH=pypath)
            if gpu is not None:
                env["CUDA_VISIBLE_DEVICES"] = str(gpu)
            env["NVSHARE_SOCK_DIR"] = str(sock_dir)
            if impl == "ours":
                env["NVSHARE_STATS_FILE"] = str(out_dir / f"engine{i}.jsonl")
            env.update({k: str(v) for k, v in (extra_env or {}).items()})
            cmd = client_cmd(spec, out_dir / f"client{i}.jsonl", f"client{i}", barrier, stop_file, seconds)
            procs.append(subprocess.Popen(cmd, env=env, cwd=ROOT, stdout=open(out_dir / f"client{i}.out", "w"),
                                          stderr=open(out_dir / f"client{i}.err", "w")))
            time.sleep(start_stagger)
        # release the clients together once each has built its inputs
        deadline = time.time() + setup_timeout
        ready = 0
        while time.time() < deadline:
            ready = 0
            for i in range(n_clients):
                f = out_dir / f"client{i}.jsonl"
                if f.exists() and '"setup_done"' in f.read_text():
                    ready += 1
            if ready == n_clients or any(p.poll() is not None for p in procs):
                break
            time.sleep(0.2)
        if ready < n_clients and all(p.poll() is None for p in procs):
            raise RuntimeError(f"only {ready} of {n_clients} clients had built their inputs after {setup_timeout} s")
        barrier.write_text("go")
        t_go = time.time()
        while any(p.poll() is None for p in procs) and time.time() - t_go < seconds + 60:
            time.sleep(1.0)
            if stop_after_handoffs and not stop_file.exists() and count_handoffs(out_dir, n_clients) >= stop_after_handoffs:
                stop_file.write_text("stop")
        if not stop_file.exists():
            stop_file.write_text("stop")
        for p in procs:
            p.wait(timeout=1800)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        stop_process(sched)
        if sock_dir.parent != out_dir:
            shutil.rmtree(sock_dir, ignore_errors=True)
    res = []
    for i, p in enumerate(procs):
        iters, meta = load_iters(out_dir / f"client{i}.jsonl") if (out_dir / f"client{i}.jsonl").exists() else ([], {})
        res.append({"rc": p.returncode, "iters": iters, "meta": meta, "out": (out_dir / f"client{i}.out").read_text()[-2000:],
                    "err_tail": (out_dir / f"client{i}.err").read_text()[-3000:]})
    return res
