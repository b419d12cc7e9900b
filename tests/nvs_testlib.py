"""Shared helpers for the test-suite: a scriptable protocol client, process
management for the daemons, and fake-driver environments."""
from __future__ import annotations

import os
import select
import signal
import socket
import struct
import subprocess
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
# NVS_TEST_BUILD points the suite at another build of the product (e.g. one made with
# -fsanitize=address,undefined: tools/sanitize.sh); NVS_TEST_PRELOAD_FIRST is put in front of
# libnvshare.so in LD_PRELOAD (the sanitizer runtime must come first)
BUILD = Path(os.environ.get("NVS_TEST_BUILD", ROOT / "nvshare_b200" / "_build"))
ORACLE = ROOT / "oracle" / "_ref"
FAKE_DIR = ORACLE / "fakecuda"
# preloaded into every reference binary: the directory NVSHARE_SOCK_DIR names instead of its fixed /var/run/nvshare
REF_SHIM = ORACLE / "libsockdir.so"

MSG_SIZE = 537
MSG_FMT = "<B254s254sQ20s"
assert struct.calcsize(MSG_FMT) == MSG_SIZE

REGISTER, SCHED_ON, SCHED_OFF, REQ_LOCK, LOCK_OK, DROP_LOCK, LOCK_RELEASED, SET_TQ = range(1, 9)
TYPE_NAMES = {1: "REGISTER", 2: "SCHED_ON", 3: "SCHED_OFF", 4: "REQ_LOCK", 5: "LOCK_OK", 6: "DROP_LOCK",
              7: "LOCK_RELEASED", 8: "SET_TQ"}


def pack(mtype, msg_id=0, data=b"", pod_name=b"", pod_namespace=b""):
    return struct.pack(MSG_FMT, mtype, pod_name, pod_namespace, msg_id, data)


def unpack(buf):
    t, pn, ns, mid, data = struct.unpack(MSG_FMT, buf)
    return {"type": t, "pod_name": pn.split(b"\0")[0], "pod_namespace": ns.split(b"\0")[0], "id": mid,
            "data": data.split(b"\0")[0], "raw_data": data}


class MockClient:
    """A scripted libnvshare stand-in speaking the 537-byte protocol."""

    def __init__(self, sock_path, name="c"):
        self.name = name
        self.s = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self.s.connect(str(sock_path))
        self.id = 1234
        self.buf = b""

    def send(self, mtype, data=b"", msg_id=None, **kw):
        self.s.sendall(pack(mtype, self.id if msg_id is None else msg_id, data, **kw))

    def send_raw(self, raw):
        self.s.sendall(raw)

    def recv(self, timeout=2.0):
        """One frame, None on timeout, b'' on EOF."""
        deadline = time.time() + timeout
        while len(self.buf) < MSG_SIZE:
            left = deadline - time.time()
            if left <= 0:
                return None
            r, _, _ = select.select([self.s], [], [], left)
            if not r:
                return None
            try:
                chunk = self.s.recv(MSG_SIZE - len(self.buf))
            except ConnectionResetError:
                return b""
            if chunk == b"":
                return b""
            self.buf += chunk
        frame, self.buf = self.buf[:MSG_SIZE], self.buf[MSG_SIZE:]
        return unpack(frame)

    def register(self, pod_name=b"none", pod_namespace=b"none"):
        self.send(REGISTER, pod_name=pod_name, pod_namespace=pod_namespace)
        m = self.recv()
        assert m not in (None, b""), "no register reply"
        self.id = int(m["data"].decode(), 16)
        return m

    def expect(self, mtype, timeout=2.0):
        m = self.recv(timeout)
        assert m not in (None, b""), f"{self.name}: expected {TYPE_NAMES[mtype]}, got {m!r}"
        assert m["type"] == mtype, f"{self.name}: expected {TYPE_NAMES[mtype]}, got {TYPE_NAMES.get(m['type'], m['type'])}"
        return m

    def expect_nothing(self, timeout=0.3):
        m = self.recv(timeout)
        assert m is None, f"{self.name}: expected silence, got {m!r}"

    def expect_closed(self, timeout=2.0):
        m = self.recv(timeout)
        assert m == b"", f"{self.name}: expected the daemon to close the connection, got {m!r}"

    def close(self):
        self.s.close()


class Daemon:
    """nvshare-scheduler (ours or the reference's) as a child process."""

    def __init__(self, impl, sock_dir: Path, debug=True, log_path=None):
        self.impl = impl
        self.sock_dir = Path(sock_dir)
        exe = (BUILD if impl == "ours" else ORACLE) / "nvshare-scheduler"
        env = dict(os.environ)
        env["NVSHARE_SOCK_DIR"] = str(self.sock_dir)
        if impl != "ours":
            env["LD_PRELOAD"] = str(REF_SHIM)
        if debug:
            env["NVSHARE_DEBUG"] = "1"
        else:
            env.pop("NVSHARE_DEBUG", None)
        self.log_path = Path(log_path) if log_path else None
        self.log = open(self.log_path, "wb") if self.log_path else subprocess.DEVNULL
        sock = self.sock_path
        if sock.exists():
            sock.unlink()
        self.p = subprocess.Popen([str(exe)], env=env, stdout=self.log, stderr=subprocess.STDOUT)
        deadline = time.time() + 5
        while not sock.exists():
            if self.p.poll() is not None or time.time() > deadline:
                raise RuntimeError(f"{impl} scheduler did not come up (rc={self.p.poll()})")
            time.sleep(0.01)
        # the socket file exists once bind() returned; listen() follows immediately
        time.sleep(0.05)

    @property
    def sock_path(self):
        return self.sock_dir / "scheduler.sock"

    def ctl(self, *args, impl=None, check=True):
        impl = impl or self.impl
        exe = (BUILD if impl == "ours" else ORACLE) / "nvsharectl"
        env = dict(os.environ, NVSHARE_SOCK_DIR=str(self.sock_dir))
        if impl != "ours":
            env["LD_PRELOAD"] = str(REF_SHIM)
        r = subprocess.run([str(exe), *args], env=env, capture_output=True, text=True)
        if check:
            assert r.returncode == 0, r.stderr
        return r

    def read_log(self):
        if not self.log_path:
            return ""
        return self.log_path.read_text(errors="replace")

    def stop(self):
        if self.p.poll() is None:
            self.p.send_signal(signal.SIGTERM)
            try:
                self.p.wait(timeout=3)
            except subprocess.TimeoutExpired:
                self.p.kill()
                self.p.wait()
        if self.log not in (None, subprocess.DEVNULL):
            self.log.close()


def fake_env(total_mib=4096, ledger=None, trace=None, devices=1, extra=None):
    """Environment for a process that should see oracle/fake_cuda.c as libcuda."""
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = str(FAKE_DIR) + (":" + env["LD_LIBRARY_PATH"] if env.get("LD_LIBRARY_PATH") else "")
    env["FAKE_CUDA_TOTAL_MIB"] = str(total_mib)
    env["FAKE_CUDA_DEVICES"] = str(devices)
    if ledger:
        env["FAKE_CUDA_LEDGER"] = str(ledger)
    if trace:
        env["FAKE_CUDA_TRACE"] = str(trace)
    if extra:
        env.update({k: str(v) for k, v in extra.items()})
    return env


def preload(lib_impl):
    if lib_impl != "ours":
        return with_ref_shim(ORACLE / "libnvshare.so")
    lib = str(BUILD / "libnvshare.so")
    first = os.environ.get("NVS_TEST_PRELOAD_FIRST")
    return f"{first}:{lib}" if first else lib


def with_ref_shim(lib):
    """LD_PRELOAD for a library that contains the reference's client code: it connects where NVSHARE_SOCK_DIR says."""
    return f"{REF_SHIM}:{lib}"
