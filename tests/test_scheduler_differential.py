"""Differential fuzz of the two daemons: the same seeded random script of client
actions (register, request, release, disconnect, nvsharectl-style status/TQ
messages, malformed frames) is applied to the REFERENCE nvshare-scheduler and to
ours; every client's received message-type sequence must be identical.  The time
quantum is set to an hour so that only message-driven transitions occur (the
timer path is covered with real time in test_scheduler_protocol.py).  What the
reference daemon did with each script is stored in
tests/golden/scheduler_differential_golden.json (tests/golden/make_golden.py)."""
from __future__ import annotations

import json
import random
import time
from pathlib import Path

import pytest

from nvs_testlib import (LOCK_RELEASED, REGISTER, REQ_LOCK, SCHED_OFF, SCHED_ON, SET_TQ, TYPE_NAMES, Daemon,
                         MockClient, pack)

GOLDEN = Path(__file__).resolve().parent / "golden" / "scheduler_differential_golden.json"
SEEDS = range(12)


def run_script(d, seed, n_clients=4, n_ops=60):
    rng = random.Random(seed)
    d.ctl("-T", "3600")
    clients = {}
    trace = {}
    log = []

    def drain():
        time.sleep(0.03)
        for name, c in list(clients.items()):
            while True:
                m = c.recv(0.01)
                if m is None:
                    break
                if m == b"":
                    trace[name].append("CLOSED")
                    c.close()
                    del clients[name]
                    break
                trace[name].append(TYPE_NAMES.get(m["type"], str(m["type"])))

    next_id = 0
    for step in range(n_ops):
        op = rng.choice(["connect", "req", "req", "req_hint", "rel", "rel", "close", "off", "on", "tq", "garbage", "unknown",
                         "req_unreg"])
        if op == "connect" or not clients:
            if len(clients) < n_clients:
                name = f"c{next_id}"
                next_id += 1
                c = MockClient(d.sock_path, name)
                clients[name] = c
                trace[name] = []
                if rng.random() < 0.85:
                    c.send(REGISTER)
                    log.append((name, "REGISTER"))
                else:
                    log.append((name, "connect-only"))
            drain()
            continue
        name = rng.choice(sorted(clients))
        c = clients[name]
        if op == "req":
            c.send(REQ_LOCK)
        elif op == "req_hint":
            # the `data` bytes of a REQ_LOCK are ours to use (the reference never reads them): whatever they hold
            # -- a need hint, an absurd one, junk -- the lock protocol itself must not change.  ('p' is excluded: a
            # pressure message is an extension that is deliberately not a lock request.)
            junk = rng.choice([b"n123", b"n0", b"n99999999999999999999", b"nabc", b"n-5", b"w3n7", b"x", b"\xff" * 19,
                               bytes(rng.randrange(1, 256) for _ in range(19))])
            if junk[:1] in (b"p", b"e"):
                junk = b"n" + junk[1:]
            c.send(REQ_LOCK, data=junk)
        elif op == "rel":
            c.send(LOCK_RELEASED)
        elif op == "close":
            c.close()
            del clients[name]
            trace[name].append("SELF-CLOSED")
        elif op == "off":
            c.send(SCHED_OFF, msg_id=0xBEEF)
        elif op == "on":
            c.send(SCHED_ON, msg_id=0xBEEF)
        elif op == "tq":
            c.send(SET_TQ, data=str(rng.choice([3600, 7200, 86400])).encode(), msg_id=0xBEEF)
        elif op == "garbage":
            c.send_raw(pack(REQ_LOCK, 1)[:rng.randint(1, 536)])
        elif op == "unknown":
            c.send(rng.randint(9, 255))
        elif op == "req_unreg":
            c.send(REGISTER)          # a second REGISTER (or a first one on a connect-only client)
        log.append((name, op))
        drain()
    drain()
    for c in clients.values():
        c.close()
    return trace, log


@pytest.mark.parametrize("seed", SEEDS)
def test_same_script_same_trace(artefacts, tmp_path, seed):
    gold = {g["seed"]: g for g in json.loads(GOLDEN.read_text())}[seed]
    want, log = gold["trace"], [tuple(x) for x in gold["script"]]
    sock_dir = tmp_path / "nvs"
    sock_dir.mkdir()
    ours = Daemon("ours", sock_dir)
    try:
        got, log2 = run_script(ours, seed)
    finally:
        ours.stop()
    assert log == log2                                    # the script itself is deterministic
    assert got == want, f"seed {seed}\nscript: {log}"
