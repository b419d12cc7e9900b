"""Parity against the committed golden fixtures (tests/golden/*.json), which
were recorded from the UNMODIFIED reference binaries by
tests/golden/make_golden.py.  These tests need neither the reference's sources nor
oracle/_ref's reference build: only our own artefacts, the fake driver and the
fixtures -- so they also run on the GPU box.

  ctl_golden.json        reference src/cli.c (+ vendored xopt): text, exit codes, frames
  hook_golden.json       reference src/hook.c: what an application sees + launch/sync pattern
  scheduler_golden.json  reference src/scheduler.c: scripted three-client scenario
"""
from __future__ import annotations

import json
import os
import socket
import subprocess
import sys
from pathlib import Path

import pytest

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "golden"))

from nvs_testlib import BUILD, MSG_SIZE, Daemon, unpack  # noqa: E402
import make_golden  # noqa: E402


def load(name):
    return json.loads((HERE / "golden" / name).read_text())


@pytest.mark.parametrize("case", load("ctl_golden.json")["daemon_down"], ids=lambda c: " ".join(c["args"]) or "noargs")
def test_ctl_text_and_exit_codes(artefacts, case, tmp_path):
    env = dict(os.environ, NVSHARE_SOCK_DIR=str(tmp_path))  # nothing listens there
    r = subprocess.run([str(BUILD / "nvsharectl"), *case["args"]], env=env, capture_output=True, text=True)
    assert r.returncode == case["rc"]
    assert r.stdout == case["stdout"]
    want = case["stderr"].replace("/var/run/nvshare/", str(tmp_path) + "/")
    assert r.stderr == want


@pytest.mark.parametrize("case", load("ctl_golden.json")["frames"], ids=lambda c: " ".join(c["args"]))
def test_ctl_frames_on_the_wire(artefacts, case, tmp_path):
    sock_path = tmp_path / "scheduler.sock"
    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    srv.bind(str(sock_path))
    srv.listen(4)
    srv.settimeout(2)
    env = dict(os.environ, NVSHARE_SOCK_DIR=str(tmp_path))
    p = subprocess.Popen([str(BUILD / "nvsharectl"), *case["args"]], env=env, stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE, text=True)
    frames = []
    try:
        while len(frames) < len(case["frames"]):
            conn, _ = srv.accept()
            conn.settimeout(2)
            buf = b""
            while len(buf) < MSG_SIZE:
                chunk = conn.recv(MSG_SIZE - len(buf))
                if not chunk:
                    break
                buf += chunk
            assert len(buf) == MSG_SIZE
            m = unpack(buf)
            frames.append({"type": m["type"], "id": m["id"], "data": m["data"].decode(),
                           "pod_name": m["pod_name"].decode(), "pod_namespace": m["pod_namespace"].decode()})
            conn.close()
    finally:
        _, se = p.communicate(timeout=5)
        srv.close()
    assert frames == case["frames"]
    assert p.returncode == case["rc"]
    assert se == case["stderr"]


def test_hook_application_view_and_sync_pattern(artefacts, tmp_path):
    """Same application, our library: identical return codes, the 1536 MiB
    reserve, the 40 GiB + 40 GiB of 80 GiB -> OUT_OF_MEMORY cap, and the reference's
    launch / cuCtxSynchronize interleaving (window 1 -> 2 -> 4)."""
    gold = load("hook_golden.json")
    sock_dir = tmp_path / "nvs"; sock_dir.mkdir()
    d = Daemon("ours", sock_dir)
    try:
        ours = make_golden.run_trace_app("ours", sock_dir, tmp_path)
    finally:
        d.stop()
    assert ours["rc"] == gold["rc"], ours["stderr"]
    assert ours["stdout"] == gold["stdout"], ours["stderr"]
    assert ours["calls"] == gold["calls"]


def test_hook_uvm_mode_matches_reference_too(artefacts, tmp_path):
    """NVSHARE_ENGINE=uvm keeps the reference's mechanism (cuMemAllocManaged)."""
    gold = load("hook_golden.json")
    sock_dir = tmp_path / "nvs"; sock_dir.mkdir()
    d = Daemon("ours", sock_dir)
    try:
        ours = make_golden.run_trace_app("ours", sock_dir, tmp_path, extra_env={"NVSHARE_ENGINE": "uvm"})
    finally:
        d.stop()
    assert ours["stdout"] == gold["stdout"], ours["stderr"]
    assert ours["calls"] == gold["calls"]
    trace = (tmp_path / "trace_ours.txt").read_text()
    assert "cuMemAllocManaged" in trace and "cuMemCreate" not in trace


def test_scheduler_scenario(artefacts, tmp_path):
    gold = load("scheduler_golden.json")
    sock_dir = tmp_path / "nvs"; sock_dir.mkdir()
    d = Daemon("ours", sock_dir)
    try:
        got = make_golden.scheduler_scenario(d)
    finally:
        d.stop()
    assert got == gold


@pytest.mark.reference
def test_fixtures_are_current(artefacts, tmp_path, default_sock_lock):
    """When the compiled reference is available, the committed hook fixture must
    still be what it produces (guards against a stale fixture)."""
    gold = load("hook_golden.json")
    fresh = make_golden.hook_golden(tmp_path)
    assert fresh == gold
