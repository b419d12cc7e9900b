"""Which GPU the idle detector watches.  The reference asks NVML for "device 0" (src/client.c:386): NVML
numbers the PHYSICAL GPUs and ignores CUDA_VISIBLE_DEVICES, so on a node with several GPUs (one scheduler per
GPU, README.md:97) every client that does not compute on physical GPU 0 watches somebody else's utilisation --
it gives its lock away while its own kernels run, or never gives it away while it idles.  Our runtime asks the
driver for the UUID of the device its application's context is on and NVML for the handle of that UUID
(client.c nvml_device_of_app); without those entry points it is the reference's device 0.
CPU only: fake driver with two "GPUs" + a fake NVML (oracle/fake_nvml.c) whose utilisation per physical GPU is
set from the environment and which records who was asked about."""
from __future__ import annotations

import subprocess

import pytest

from nvs_testlib import ORACLE, Daemon, fake_env, preload

FAKE_NVML = ORACLE / "fakenvml"


def run_idle_client(sock_dir, tmp_path, util, extra=None):
    env = fake_env(total_mib=400, ledger=tmp_path / "hbm", devices=2,
                   extra={"NVSHARE_HOST_ARENA_MIB": 64, "NVSHARE_CHUNK_MIB": 8, "NVSHARE_DEBUG": 1, "NVSHARE_SOCK_DIR": sock_dir,
                          "NVSHARE_POOL": "private", "FAKE_CUDA_DEVICE": 1, "FAKE_NVML_UTIL": util,
                          "FAKE_NVML_TRACE": tmp_path / "nvml.trace", **(extra or {})})
    env["LD_LIBRARY_PATH"] = f"{FAKE_NVML}:{env['LD_LIBRARY_PATH']}"
    env["LD_PRELOAD"] = preload("ours")
    d = Daemon("ours", sock_dir)
    try:
        d.ctl("-T", "30")
        # 3 x 16 MiB, one second of work, then 7 s idle holding the lock (the detector looks every 5 s), then verify
        r = subprocess.run([str(ORACLE / "driver_app"), "16", "1.0", "1", "3", "7.0"], env=env, capture_output=True, text=True,
                           timeout=120)
    finally:
        d.stop()
    assert r.returncode == 0 and "RESULT PASS" in r.stdout, r.stdout + r.stderr[-2500:]
    trace = (tmp_path / "nvml.trace").read_text().split("\n") if (tmp_path / "nvml.trace").exists() else []
    return r.stderr, [l for l in trace if l]


def test_idle_client_on_gpu1_releases_although_gpu0_is_busy(artefacts, sock_dir, tmp_path):
    err, trace = run_idle_client(sock_dir, tmp_path, "100,0")           # physical GPU 0 busy, GPU 1 (ours) idle
    assert "Found NVML" in err
    h = (b"GPU-FAKE-H100-" + bytes([0, 1])).hex()                        # the fake driver's UUID of physical GPU 1
    assert f"Early release watches the utilisation of GPU-{h[:8]}-{h[8:12]}-{h[12:16]}-{h[16:20]}-{h[20:]} (CUDA device 1)" in err
    assert "by_uuid 1" in trace and "util 1" in trace and "util 0" not in trace
    assert "Releasing the lock early due to inactivity" in err


def test_busy_client_on_gpu1_keeps_its_lock_although_gpu0_is_idle(artefacts, sock_dir, tmp_path):
    err, trace = run_idle_client(sock_dir, tmp_path, "0,100")           # GPU 0 idle, ours busy (work submitted earlier)
    assert "util 1" in trace and "util 0" not in trace
    assert "Early release timer elapsed but we are not idle" in err
    assert "Releasing the lock early due to inactivity" not in err


def test_without_uuid_lookup_it_is_the_references_device_0(artefacts, sock_dir, tmp_path):
    err, trace = run_idle_client(sock_dir, tmp_path, "0,100", extra={"FAKE_NVML_NO_UUID": 1})
    assert "watching NVML device 0 like the reference" in err
    assert "by_index 0" in trace and "util 0" in trace and "util 1" not in trace
    assert "Releasing the lock early due to inactivity" in err          # (GPU 0 is idle: the reference's answer)
