"""INTEGRATION.md section B on the real driver: the unmodified reference hook.c + client.c with the binding of that
section (oracle/bind_reference.py; built beside the reference when its sources are present, travels as
oracle/_ref/libnvshare_bound.so) and our libnvs_engine.so behind it, under the REFERENCE daemon.  Two driver-API
clients that only copy (every copy entry point is in the reference's gated set; its hook knows nothing about
memsets or cuLaunchKernelEx, which a VMM-backed allocation would need gated too): with the reference daemon
every hand-off swaps everything out and in again through nvs_evict / nvs_fetch_all, and the payload that went
round the buffers must come back word for word.  (Sorted last: written after the round's GPU minutes were spent;
the same test runs on the fake driver in tests/test_bound_reference.py.)"""
from __future__ import annotations

import json
import os
import re
import subprocess

import pytest

from nvs_testlib import ORACLE, Daemon, with_ref_shim

pytestmark = [pytest.mark.gpu, pytest.mark.reference]
BOUND = ORACLE / "libnvshare_bound.so"


def test_reference_hook_and_client_over_our_engine_on_the_gpu(artefacts, default_sock_lock, tmp_path):
    if not BOUND.exists():
        pytest.skip("oracle/_ref/libnvshare_bound.so was not built (reference sources absent at build time)")
    d = Daemon("reference", default_sock_lock, log_path=tmp_path / "sched.log")
    try:
        procs = []
        d.ctl("-T", "1")
        for i in (1, 2):
            env = dict(os.environ, LD_PRELOAD=with_ref_shim(BOUND), NVSHARE_DEBUG="1", DRIVER_APP_NO_LAUNCH="1",
                       NVSHARE_STATS_FILE=str(tmp_path / f"stats{i}.jsonl"))
            procs.append(subprocess.Popen([str(ORACLE / "driver_app"), "256", "6.0", str(i), "3"], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        outs = [p.communicate(timeout=300) for p in procs]
    finally:
        for p in procs:                     # (a client that is still there after a failure must not outlive the test)
            if p.poll() is None:
                p.kill()
        d.stop()
    for i, (p, (out, err)) in enumerate(zip(procs, outs), 1):
        assert p.returncode == 0 and re.search(r"RESULT PASS iters=\d+ mismatches=0", out), out + err[-2500:]
        recs = [json.loads(l) for l in (tmp_path / f"stats{i}.jsonl").read_text().splitlines()]
        ev = [r for r in recs if r["op"] == "evict"]
        assert ev and sum(r["bytes"] + r.get("clean_bytes", 0) + r.get("elided_bytes", 0) for r in ev) >= 768 << 20
        assert [r for r in recs if r["op"] == "fetch"]
