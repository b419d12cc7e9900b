#!/usr/bin/env python3
"""Regenerate tests/golden/*.json from the UNMODIFIED reference binaries in
oracle/_ref (built by oracle/Makefile where the reference's sources are
present; oracle/_ref/libsockdir.so lets them use a temporary socket directory
instead of their fixed /var/run/nvshare):

    python tests/golden/make_golden.py

The fixtures pin what the reference *does* (not what its source seems to say):
  ctl_golden.json        nvsharectl: stdout/stderr/exit code per argument list with
                         the daemon down, and the exact 537-byte frames it sends
                         when something is listening
  hook_golden.json       libnvshare.so under a fake CUDA driver: what the
                         application observes (return codes, reserve) and the
                         filtered driver-call trace (launch / sync pattern)
  scheduler_golden.json  a scripted three-client scenario: which message types
                         each client receives, in order
  reference_exports.json the driver entry points (and dlsym) libnvshare.so exports
  workload_checksums.json
                         float64 checksums of the output of the seeded add / matmul
                         workloads of tests/test_gpu_hooked.py, run un-hooked on an
                         H100 (`--checksums`, needs a GPU; not written by a plain run).
                         The reference's library changes where the bytes live, not
                         what they are: these are the values its arm must reproduce
  scheduler_differential_golden.json
                         the seeded scripts of tests/test_scheduler_differential.py:
                         what each client received from the reference daemon
The reference pins no numerical result for the data path (its tests print PASS
unconditionally), so there is no data fixture from it; data parity is defined
in tests/ against oracle/nvshare_oracle.c.
"""
from __future__ import annotations

import json
import os
import socket
import subprocess
import sys
import time
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT))

from nvs_testlib import (DROP_LOCK, LOCK_OK, LOCK_RELEASED, MSG_SIZE, ORACLE, REF_SHIM, REQ_LOCK, TYPE_NAMES,  # noqa: E402
                         Daemon, MockClient, fake_env, preload, unpack)

CHECKSUM_WORKLOADS = (("add", 12000), ("matmul", 6144))

CTL_ARGS = [[], ["-h"], ["--help"], ["-S", "maybe"], ["-T", "-3"], ["--bogus"], ["-x"], ["foo"], ["-T", "abc"],
            ["-T", "0"], ["-T"], ["-S"], ["-T5"], ["--help=1"], ["-hT"], ["--set-tq=abc"], ["--anti-thrash"],
            ["-T", "1.5"], ["-T", "5"], ["--set-tq=7"]]


def ctl_golden(sock_dir):
    exe = ORACLE / "nvsharectl"
    env = dict(os.environ, NVSHARE_SOCK_DIR=str(sock_dir), LD_PRELOAD=str(REF_SHIM))
    out = {"daemon_down": [], "frames": []}
    sock_path = Path(sock_dir) / "scheduler.sock"
    if sock_path.exists():
        sock_path.unlink()
    for args in CTL_ARGS:
        r = subprocess.run([str(exe), *args], env=env, capture_output=True, text=True)
        out["daemon_down"].append({"args": args, "rc": r.returncode, "stdout": r.stdout, "stderr": r.stderr})
    # a listener that just records frames
    os.makedirs(sock_path.parent, exist_ok=True)
    for args in (["-T", "5"], ["--set-tq=7"], ["-S", "on"], ["-S", "off"], ["-S", "off", "-T", "9"]):
        if sock_path.exists():
            sock_path.unlink()
        srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        srv.bind(str(sock_path))
        srv.listen(4)
        srv.settimeout(2)
        p = subprocess.Popen([str(exe), *args], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        frames = []
        try:
            while True:
                conn, _ = srv.accept()
                buf = b""
                conn.settimeout(2)
                while len(buf) < MSG_SIZE:
                    chunk = conn.recv(MSG_SIZE - len(buf))
                    if not chunk:
                        break
                    buf += chunk
                m = unpack(buf)
                frames.append({"type": m["type"], "id": m["id"], "data": m["data"].decode(),
                               "pod_name": m["pod_name"].decode(), "pod_namespace": m["pod_namespace"].decode()})
                conn.close()
        except socket.timeout:
            pass
        so, se = p.communicate(timeout=5)
        srv.close()
        out["frames"].append({"args": args, "rc": p.returncode, "stderr": se, "frames": frames})
    if sock_path.exists():
        sock_path.unlink()
    return out


FILTER = ("cuInit", "cuLaunchKernel", "cuCtxSynchronize", "cuMemcpyHtoD", "cuMemcpyDtoH")


def run_trace_app(lib_impl, sched_dir, tmp, alloc_mib=40 * 1024, total_mib=80 * 1024, extra_env=None):
    trace = Path(tmp) / f"trace_{lib_impl}.txt"
    if trace.exists():
        trace.unlink()
    env = fake_env(total_mib=total_mib, trace=trace, extra=extra_env)
    env["LD_PRELOAD"] = preload(lib_impl)
    env["NVSHARE_SOCK_DIR"] = str(sched_dir)
    r = subprocess.run([str(ORACLE / "trace_app"), str(alloc_mib), "3"], env=env, capture_output=True, text=True,
                       timeout=120)
    # the engine's own kernels (background pre-cleaning, scans) are not the application's calls
    names = [ln.split()[0] for ln in trace.read_text().splitlines()
             if ln.split() and not (len(ln.split()) > 1 and ln.split()[1].startswith("nvs_slab"))]
    # The real cuMemFree (what the reference's hook calls) synchronises INSIDE the driver, where no trace
    # sees it; our engine frees VMM memory with cuMemUnmap, which does not, so it drains the context
    # itself first.  That explicit call stands for the implicit one and is not part of the comparison.
    calls = [n for i, n in enumerate(names)
             if n in FILTER and not (n == "cuCtxSynchronize" and i + 1 < len(names) and names[i + 1] == "cuMemUnmap")]
    return {"rc": r.returncode, "stdout": r.stdout.splitlines(), "calls": calls, "stderr": r.stderr}


def fresh_dir(tmp, name):
    d = Path(tmp) / name
    d.mkdir()
    return d


def hook_golden(tmp):
    d = Daemon("reference", fresh_dir(tmp, "hook"))
    try:
        g = run_trace_app("reference", d.sock_dir, tmp)
    finally:
        d.stop()
    g.pop("stderr")
    return g


def scheduler_scenario(d):
    """Three clients, TQ=1: returns {client: [message type names received]}."""
    d.ctl("-T", "1")
    cs = {n: MockClient(d.sock_path, n) for n in "abc"}
    got = {n: [] for n in cs}
    for c in cs.values():
        got[c.name].append(TYPE_NAMES[c.register()["type"]])
    for n in "abc":
        cs[n].send(REQ_LOCK)
        time.sleep(0.05)
    deadline = time.time() + 6
    released = set()
    while time.time() < deadline and len(released) < 3:
        for n, c in cs.items():
            m = c.recv(0.05)
            if m in (None, b""):
                continue
            got[n].append(TYPE_NAMES[m["type"]])
            if m["type"] == DROP_LOCK:
                c.send(LOCK_RELEASED)
                released.add(n)
    for c in cs.values():
        c.close()
    return got


def exports_golden():
    out = subprocess.run(["nm", "-D", "--defined-only", str(ORACLE / "libnvshare.so")], capture_output=True, text=True,
                         check=True).stdout
    syms = {ln.split()[-1].split("@")[0] for ln in out.splitlines() if ln.strip()}
    return sorted(s for s in syms if s == "dlsym" or (s[:2] == "cu" and s[2:3].isupper()))


def differential_golden(tmp):
    from test_scheduler_differential import SEEDS, run_script
    out = []
    for seed in SEEDS:
        d = Daemon("reference", fresh_dir(tmp, f"diff{seed}"))
        try:
            trace, log = run_script(d, seed)
        finally:
            d.stop()
        out.append({"seed": seed, "script": [list(x) for x in log], "trace": trace})
    return out


def workload_checksums_golden():
    out = {}
    for kind, n in CHECKSUM_WORKLOADS:
        env = dict(os.environ, PYTHONPATH=str(ROOT))
        env.pop("LD_PRELOAD", None)
        r = subprocess.run([sys.executable, "-m", "nvshare_b200.workloads", "--kind", kind, "--n", str(n), "--iters", "1000000",
                            "--seconds", "6", "--pattern", "pos"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
        if r.returncode != 0 or not r.stdout.startswith("PASS"):
            sys.exit(f"un-hooked {kind} n={n} failed:\n{r.stdout}{r.stderr[-3000:]}")
        summary = json.loads(r.stdout.splitlines()[0].split(" ", 1)[1])
        out[f"{kind}_{n}"] = [summary["z_sum"], summary["z_wsum"]]
    return out


def scheduler_golden(tmp):
    d = Daemon("reference", fresh_dir(tmp, "scenario"))
    try:
        return scheduler_scenario(d)
    finally:
        d.stop()


def main():
    import tempfile
    if "--checksums" in sys.argv:
        json.dump(workload_checksums_golden(), open(HERE / "workload_checksums.json", "w"), indent=1)
        return
    if not (ORACLE / "nvshare-scheduler").exists():
        sys.exit("oracle/_ref is not built; run `make -C oracle` where the reference's sources are")
    with tempfile.TemporaryDirectory(dir="/tmp") as tmp:
        json.dump(ctl_golden(fresh_dir(tmp, "ctl")), open(HERE / "ctl_golden.json", "w"), indent=1)
        json.dump(hook_golden(tmp), open(HERE / "hook_golden.json", "w"), indent=1)
        json.dump(scheduler_golden(tmp), open(HERE / "scheduler_golden.json", "w"), indent=1)
        json.dump(exports_golden(), open(HERE / "reference_exports.json", "w"), indent=1)
        json.dump(differential_golden(tmp), open(HERE / "scheduler_differential_golden.json", "w"), indent=1)
    print("wrote", [p.name for p in HERE.glob("*.json")])


if __name__ == "__main__":
    main()
