"""Clean-slab skip (SURVEY 8f rank 3, "pre-cleaning"): backing copies are kept
after a fetch, every slab's 128-bit content hash is recorded when its copy is
written, and the next eviction copies only slabs whose hash changed.  CPU, fake
driver (which computes the same hash as the sm_90a scan kernel through
oracle/slab_hash_ref.h); the kernel itself is checked against the oracle on the
GPU (tests/test_gpu_engine.py)."""
from __future__ import annotations

import ctypes as C
import struct
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from nvs_testlib import FAKE_DIR, ORACLE, ROOT

MiB = 1 << 20
SLAB = 2 * MiB


@pytest.fixture(scope="module")
def fake(artefacts):
    lib = C.CDLL(str(FAKE_DIR / "libcuda.so.1"), mode=C.RTLD_GLOBAL)
    lib.fake_cuda_phys_used.restype = C.c_uint64
    assert lib.cuInit(0) == 0
    ctx = C.c_void_p()
    assert lib.cuDevicePrimaryCtxRetain(C.byref(ctx), 0) == 0
    assert lib.cuCtxSetCurrent(ctx) == 0
    return lib


@pytest.fixture(scope="module")
def oracle(artefacts):
    lib = C.CDLL(str(ORACLE / "liboracle.so"))
    lib.oracle_slab_hash.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64 * 2)]
    return lib


def view(ptr, nbytes):
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def mk(**kw):
    from nvshare_b200 import engine as E
    # background pre-cleaning is tested on its own below: with it the byte counts asserted here depend on timing
    args = dict(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, batch_bytes=24 * MiB, oom_wait_ms=300, prepin=0, preclean=0)
    args.update(kw)
    return E.Engine(**args)


def test_unchanged_data_is_not_copied_again(fake):
    e = mk()
    try:
        p = e.alloc(48 * MiB)
        e.fetch_all()
        e.pattern_fill(p, 48 * MiB // 8, seed=7)
        r1 = e.evict(0)
        assert r1["bytes"] == 48 * MiB and r1["clean_bytes"] == 0
        e.fetch_all()
        st = e.stats()
        assert st["retained_bytes"] == 48 * MiB and st["host_pool_used"] == 48 * MiB      # the copies stay
        r2 = e.evict(0)
        assert r2["bytes"] == 0 and r2["clean_bytes"] == 48 * MiB and r2["ce_calls"] == 0  # nothing crosses the link
        assert e.stats()["swapped_bytes"] == 48 * MiB
        f = e.fetch_all()
        assert f["bytes"] == 48 * MiB
        assert e.pattern_verify(p, 48 * MiB // 8, seed=7) == 0
        assert e.stats()["clean_skipped_bytes_total"] == 48 * MiB
        e.free(p)
        assert e.stats()["host_pool_used"] == 0 and e.stats()["retained_bytes"] == 0
    finally:
        e.close()


def test_one_changed_word_is_seen_after_a_round_trip(fake):
    """The VERDICT's test: mutate one word in a "clean" slab; it must survive the hand-off."""
    e = mk()
    try:
        p = e.alloc(32 * MiB)
        e.fetch_all()
        e.pattern_fill(p, 32 * MiB // 8, seed=3)
        e.evict(0); e.fetch_all()
        words = view(p, 32 * MiB).view(np.uint64)
        before = words.copy()
        words[(10 * MiB) // 8 + 12345] ^= 1                  # one bit, slab 5 (chunk 1)
        r = e.evict(0)
        assert r["bytes"] == SLAB and r["clean_bytes"] == 32 * MiB - SLAB        # that slab, and only that one
        e.fetch_all()
        after = view(p, 32 * MiB).view(np.uint64)
        before[(10 * MiB) // 8 + 12345] ^= 1
        assert np.array_equal(after, before)
        e.free(p)
    finally:
        e.close()


def test_retention_off_moves_everything_every_time(fake):
    e = mk(retain=0)
    try:
        p = e.alloc(16 * MiB)
        e.fetch_all()
        e.pattern_fill(p, 16 * MiB // 8, seed=5)
        e.evict(0); e.fetch_all()
        assert e.stats()["host_pool_used"] == 0              # round-1 behaviour: backing released at fetch
        r = e.evict(0)
        assert r["bytes"] == 16 * MiB and r["clean_bytes"] == 0
        e.fetch_all(); e.free(p)
    finally:
        e.close()


def test_partial_eviction_prefers_clean_chunks(fake):
    """What is out never costs a miss later (everything must be resident to run): victims are
    the chunks that are cheapest to put out -- the ones whose kept copy is still valid."""
    e = mk()
    try:
        a = e.alloc(16 * MiB)                                # low addresses, rewritten every "iteration"
        b = e.alloc(16 * MiB)                                # never changes
        e.fetch_all()
        e.pattern_fill(a, 16 * MiB // 8, seed=1)
        e.pattern_fill(b, 16 * MiB // 8, seed=2)
        e.evict(0); e.fetch_all()
        e.pattern_fill(a, 16 * MiB // 8, seed=11)            # a is dirty now
        r = e.evict(12 * MiB)                                # two 8 MiB chunks needed
        assert r["bytes"] == 0 and r["clean_bytes"] == 16 * MiB          # b went out for free; a stayed
        st = e.stats()
        assert st["resident_bytes"] == 16 * MiB and st["retained_bytes"] == 16 * MiB
        e.fetch_all()
        assert e.pattern_verify(a, 16 * MiB // 8, seed=11) == 0 and e.pattern_verify(b, 16 * MiB // 8, seed=2) == 0
        e.free(a); e.free(b)
    finally:
        e.close()


def test_recently_written_chunks_are_evicted_last(fake):
    """VERDICT #9: a hot low-address allocation survives a partial eviction (nvs_touch is what the
    hook calls for cuMemcpy* / cuMemset* destinations)."""
    e = mk(retain=0, elide_constant=0)
    try:
        hot = e.alloc(16 * MiB)                              # lowest addresses
        cold = e.alloc(32 * MiB)
        e.fetch_all()
        e.touch(hot, 16 * MiB)
        r = e.evict(16 * MiB)
        assert r["bytes"] == 16 * MiB
        # the hot allocation is still on the GPU: it can be written without faulting (fake driver: SIGSEGV)
        view(hot, 16 * MiB)[:] = 1
        st = e.stats()
        assert st["resident_bytes"] == 32 * MiB
        e.fetch_all(); e.free(hot); e.free(cold)
    finally:
        e.close()


def test_volatile_chunks_stop_being_retained(fake):
    e = mk()
    try:
        p = e.alloc(8 * MiB)
        e.fetch_all()
        for i in range(4):
            e.pattern_fill(p, 8 * MiB // 8, seed=100 + i)    # changes completely between hand-offs
            r = e.evict(0)
            assert r["bytes"] == 8 * MiB
            e.fetch_all()
        # after it was found dirty against a kept copy, the copy is given back at fetch
        assert e.stats()["retained_bytes"] == 0 and e.stats()["host_pool_used"] == 0
        assert e.pattern_verify(p, 8 * MiB // 8, seed=103) == 0
        e.free(p)
    finally:
        e.close()


def test_private_pool_takes_over_kept_copies_before_it_grows(fake):
    e = mk(host_arena_bytes=32 * MiB)
    try:
        a = e.alloc(24 * MiB); e.fetch_all(); e.pattern_fill(a, 24 * MiB // 8, seed=1)
        e.evict(0); e.fetch_all()                            # a resident, 24 MiB of copies kept
        b = e.alloc(24 * MiB)                                # resident mode: mapped at once
        e.pattern_fill(b, 24 * MiB // 8, seed=2)
        e.pattern_fill(a, 24 * MiB // 8, seed=3)             # a's copies are stale now ...
        e.touch(a, 24 * MiB)                                 # ... and a was written last: b goes first
        r = e.evict(24 * MiB)                                # b needs 24 MiB of units: 8 free + 16 taken over from a
        assert r["bytes"] == 24 * MiB
        st = e.stats()
        assert st["host_pool_bytes"] == 32 * MiB             # no second arena was pinned
        assert st["stolen_slabs_total"] >= 8 and st["resident_bytes"] == 24 * MiB
        e.fetch_all()
        assert e.pattern_verify(a, 24 * MiB // 8, seed=3) == 0 and e.pattern_verify(b, 24 * MiB // 8, seed=2) == 0
        r = e.evict(0)                                       # a lost (part of) its copies: it moves again
        assert r["bytes"] + r["clean_bytes"] == 48 * MiB and r["bytes"] >= 24 * MiB
        e.fetch_all()
        assert e.pattern_verify(a, 24 * MiB // 8, seed=3) == 0 and e.pattern_verify(b, 24 * MiB // 8, seed=2) == 0
        e.free(a); e.free(b)
    finally:
        e.close()


def test_host_io_invalidates_the_recorded_hash(fake):
    """A lock-free upload changes the backing copy under its hash; if the application then
    restores the old contents on the GPU the slab must NOT be taken for clean."""
    e = mk()
    try:
        p = e.alloc(8 * MiB); e.fetch_all(); e.pattern_fill(p, 8 * MiB // 8, seed=9)
        old = view(p, 8 * MiB).copy()
        e.evict(0)
        new = np.full(SLAB, 0x5A, dtype=np.uint8)
        assert e.host_io(p, new.ctypes.data, SLAB, True) == 0        # overwrite slab 0 in the backing copy
        e.fetch_all()
        assert np.array_equal(view(p, SLAB), new)
        view(p, SLAB)[:] = old[:SLAB]                                 # back to the old contents (old hash)
        r = e.evict(0)
        assert r["bytes"] == SLAB                                     # copied all the same
        e.fetch_all()
        assert np.array_equal(view(p, 8 * MiB), old)
        e.free(p)
    finally:
        e.close()


def test_scan_slabs_matches_the_oracle_hash(fake, oracle):
    e = mk()
    try:
        rng = np.random.default_rng(3)
        buf = rng.integers(0, 256, 3 * SLAB + 4096, dtype=np.uint8)
        base = (buf.ctypes.data + 15) & ~15
        descs = [(base, 0, SLAB), (base + SLAB, 0, SLAB), (base + 2 * SLAB, 0, 4096 + 16)]
        from nvshare_b200 import engine as E
        out = E.scan_slabs(e, descs, want_hash=True)
        for (src, _, n), o in zip(descs, out):
            want = (C.c_uint64 * 2)()
            oracle.oracle_slab_hash(src, n, C.byref(want))
            assert (o["h0"], o["h1"]) == (want[0], want[1]) and o["is_const"] == 0
        flip = view(base + 7 * 4096 + 3, 1)
        flip[0] ^= 0x10
        again = E.scan_slabs(e, descs[:1], want_hash=True)[0]
        assert (again["h0"], again["h1"]) != (out[0]["h0"], out[0]["h1"])
        nohash = E.scan_slabs(e, descs[:1], want_hash=False)[0]
        assert nohash["h0"] == 0 and nohash["h1"] == 0
    finally:
        e.close()


def test_background_precleaning_through_the_c_abi(fake):
    """The owner holds the lock (resident mode) and leaves its data alone: the pre-cleaner writes every resident
    chunk back with the fused copy + hash kernel; the eviction that follows copies only what changed after that."""
    import time
    e = mk(preclean=1, prepin=1)                         # the pre-cleaner only takes units that are already pinned
    try:
        p = e.alloc(32 * MiB)
        e.fetch_all()
        # fetch_all already puts the engine in resident mode: the pre-cleaner may write chunks back before the fill
        # below (it waits for the fill, and the fill for it).  Such a copy holds the old contents, so the eviction
        # copies that chunk again.  It takes chunks in allocation order, and each one once per residency.
        before = e.stats()["precleaned_bytes_total"]
        e.pattern_fill(p, 32 * MiB // 8, seed=77)
        after = e.stats()["precleaned_bytes_total"]
        e.set_resident_mode(True)                            # what libnvshare.so says when LOCK_OK has been handled
        deadline = time.time() + 10
        while e.stats()["precleaned_bytes_total"] < 32 * MiB and time.time() < deadline:
            time.sleep(0.02)
        st = e.stats()
        assert st["precleaned_bytes_total"] >= 32 * MiB and st["retained_bytes"] == 32 * MiB
        view(p + 5 * MiB, 8)[:] = 1                          # ... then one slab changes after all
        r = e.evict(0)
        # stale: the first k chunks, written back before the fill; the changed slab lies in chunk 0
        stale = [max(k, SLAB) for k in range(before, after + 1, 8 * MiB)]
        assert r["bytes"] in stale and r["clean_bytes"] == 32 * MiB - r["bytes"], (r, before, after)
        e.fetch_all()
        want = np.empty(32 * MiB // 8, dtype=np.uint64)
        C.CDLL(str(ORACLE / "liboracle.so")).oracle_pattern_fill(C.c_void_p(want.ctypes.data), C.c_uint64(want.size), C.c_uint64(0), C.c_uint64(77))
        want.view(np.uint8)[5 * MiB:5 * MiB + 8] = 1
        assert np.array_equal(view(p, 32 * MiB).view(np.uint64), want)
        e.free(p)
    finally:
        e.close()


def test_shared_pool_other_client_takes_over_kept_copies(artefacts, tmp_path):
    """Two clients, one shared pool that cannot hold what both would like to keep: the second
    takes over the first one's kept (reclaimable) units; the first notices at its next eviction
    and moves everything again; nobody loses data."""
    pool = tmp_path / "pool"
    prelude = textwrap.dedent(f"""
        import ctypes as C, os, sys, time
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        MiB = 1 << 20
        e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=32 * MiB, shared_pool_path={str(pool)!r},
                     shared_pool_bytes=64 * MiB, prepin=0, oom_wait_ms=2000, preclean=0)
        step = {str(tmp_path)!r} + "/step"
        def wait(n):
            while not os.path.exists(step + str(n)): time.sleep(0.01)
        def done(n):
            open(step + str(n), "w").close()
    """)
    a_code = prelude + textwrap.dedent("""
        p = e.alloc(48 * MiB); e.fetch_all(); e.pattern_fill(p, 48 * MiB // 8, seed=1)
        e.evict(0); e.fetch_all()                      # 48 MiB of kept copies in a 64 MiB pool
        print("A_RETAINED", e.stats()["retained_bytes"] // MiB, flush=True)
        done(1); wait(2)                               # B evicts 40 MiB meanwhile
        r = e.evict(0)
        print("A_EVICT", r["bytes"] // MiB, r["clean_bytes"] // MiB, flush=True)
        e.fetch_all(); print("A_BAD", e.pattern_verify(p, 48 * MiB // 8, seed=1), flush=True)
        e.free(p); e.close()
    """)
    b_code = prelude + textwrap.dedent("""
        wait(1)
        q = e.alloc(40 * MiB); e.fetch_all(); e.pattern_fill(q, 40 * MiB // 8, seed=2)
        r = e.evict(0)                                 # 16 MiB free + 24 MiB taken over from A
        print("B_EVICT", r["bytes"] // MiB, e.stats()["stolen_slabs_total"], flush=True)
        e.fetch_all(); print("B_BAD", e.pattern_verify(q, 40 * MiB // 8, seed=2), flush=True)
        e.free(q); e.close()
        done(2)
    """)
    env = dict(__import__("os").environ, FAKE_CUDA_TOTAL_MIB="512")
    pa = subprocess.Popen([sys.executable, "-c", a_code], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    pb = subprocess.Popen([sys.executable, "-c", b_code], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    oa, ea = pa.communicate(timeout=60)
    ob, eb = pb.communicate(timeout=60)
    assert pa.returncode == 0 and pb.returncode == 0, oa + ea + ob + eb
    assert "A_RETAINED 48" in oa and "A_BAD 0" in oa and "B_BAD 0" in ob, oa + ob
    assert "B_EVICT 40 12" in ob, ob                           # 12 slabs = 24 MiB taken over
    moved, clean = map(int, oa.split("A_EVICT")[1].split()[:2])
    assert moved + clean == 48 and 24 <= moved <= 48, oa       # chunks that lost units are copied again in full
    used = struct.unpack("<QIIQQ", pool.open("rb").read(32))[4]
    assert used == 0
