"""Host logic of the swap engine (nvshare_b200/csrc/engine.c) through its C-ABI
(include/nvshare_engine.h), on CPU against oracle/fake_cuda.c.  The fake driver
executes the copy kernels' byte semantics, so these tests cover descriptor
generation, chunk state machine, LRU order, pools and error paths -- NOT the
CUDA kernels themselves (tests/test_gpu_*.py do that on an H100).

Checker: oracle/nvshare_oracle.c (liboracle.so) -- oracle_slab_move,
oracle_pattern_*.
"""
from __future__ import annotations

import ctypes as C
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
    lib.oracle_pattern.restype = C.c_uint64
    lib.oracle_pattern.argtypes = [C.c_uint64, C.c_uint64]
    lib.oracle_pattern_fill.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    lib.oracle_pattern_mismatches.restype = C.c_uint64
    lib.oracle_pattern_mismatches.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    lib.oracle_slab_move.argtypes = [C.c_void_p, C.c_uint32]
    return lib


@pytest.fixture()
def engine(fake):
    from nvshare_b200 import engine as E
    # elision off: most tests below move freshly mapped (all-zero) memory on purpose
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, batch_bytes=24 * MiB, oom_wait_ms=300,
                 elide_constant=0, retain=0)
    yield e
    e.close()


def view(ptr, nbytes):
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def test_version_and_default_config(fake):
    from nvshare_b200 import engine as E
    assert b"sm_90a" in E.load().nvs_engine_version()
    cfg = E.default_config()
    assert cfg.chunk_bytes == 256 * MiB and cfg.host_arena_bytes == 1024 * MiB
    # pinned-host tier on the copy engines (256-byte TLPs), peer tier on the sm_90a kernel: engine.c, probes D/G
    assert cfg.evict_variant == E.COPY_CE and cfg.fetch_variant == E.COPY_CE
    assert cfg.peer_evict_variant == E.COPY_TMA and cfg.peer_fetch_variant == E.COPY_CE and cfg.retain == 1
    assert cfg.tma_stages == 6 and cfg.tma_tile_bytes == 32768 and cfg.tma_warps == 1


def test_alloc_is_virtual_until_fetched(engine, fake):
    base = fake.fake_cuda_phys_used()
    p = engine.alloc(20 * MiB + 5)           # rounds up to 22 MiB of VA: 3 chunks of 8+8+6
    st = engine.stats()
    assert st["va_bytes"] == 22 * MiB and st["unbacked_bytes"] == 22 * MiB and st["resident_bytes"] == 0
    assert fake.fake_cuda_phys_used() == base
    rep = engine.fetch_all()
    assert rep["chunks"] == 3 and rep["bytes"] == 0          # nothing to copy for fresh memory
    assert fake.fake_cuda_phys_used() == base + 22 * MiB
    assert engine.stats()["resident_bytes"] == 22 * MiB
    engine.free(p)
    assert fake.fake_cuda_phys_used() == base


def test_round_trips_are_bit_exact_against_oracle(engine, fake, oracle):
    sizes = [2 * MiB, 7 * MiB, 8 * MiB, 33 * MiB]            # single slab, ragged, exact chunk, multi-chunk
    ptrs = [engine.alloc(s) for s in sizes]
    engine.fetch_all()
    for k, (p, s) in enumerate(zip(ptrs, sizes)):
        engine.pattern_fill(p, s // 8, first_index=k << 32, seed=42 + k)
    for cycle in range(3):
        rep = engine.evict(0)
        assert rep["bytes"] == sum((s + SLAB - 1) // SLAB * SLAB for s in sizes)
        assert engine.stats()["resident_bytes"] == 0
        rep = engine.fetch_all()
        assert rep["bytes"] == sum((s + SLAB - 1) // SLAB * SLAB for s in sizes)
        for k, (p, s) in enumerate(zip(ptrs, sizes)):
            # checker 1: the oracle's own pattern check on the raw bytes
            assert oracle.oracle_pattern_mismatches(p, s // 8, k << 32, 42 + k) == 0
            # checker 2: the engine's verify kernel agrees
            assert engine.pattern_verify(p, s // 8, first_index=k << 32, seed=42 + k) == 0
    # the oracle would notice a swapped pair of slabs
    a = view(ptrs[3], 4 * MiB).copy()
    view(ptrs[3], 2 * MiB)[:] = a[2 * MiB:]
    view(ptrs[3] + 2 * MiB, 2 * MiB)[:] = a[:2 * MiB]
    assert oracle.oracle_pattern_mismatches(ptrs[3], sizes[3] // 8, 3 << 32, 45) > 0
    for p in ptrs:
        engine.free(p)


@pytest.mark.parametrize("variant", ["tma", "ldg", "ce"])
def test_copy_slabs_matches_oracle_move(engine, oracle, variant):
    rng = np.random.default_rng(7)
    n, size = 9, 3 * SLAB
    src = np.frombuffer(rng.bytes(size), dtype=np.uint8).copy()
    dst_eng = np.zeros(size, dtype=np.uint8)
    dst_orc = np.zeros(size, dtype=np.uint8)
    # ragged descriptors: 16-byte multiples, shuffled, non-overlapping
    cuts = sorted(set([0, size] + [int(x) & ~15 for x in rng.integers(16, size - 16, n - 1)]))
    pieces = [(cuts[i], cuts[i + 1] - cuts[i]) for i in range(len(cuts) - 1) if cuts[i + 1] - cuts[i] <= SLAB]
    rng.shuffle(pieces)
    from nvshare_b200.engine import CopyDesc
    descs = [(src.ctypes.data + off, dst_eng.ctypes.data + off, ln) for off, ln in pieces]
    ms = engine.copy_slabs(descs, variant=variant, grid=4)
    assert ms > 0
    arr = (CopyDesc * len(pieces))()
    for i, (off, ln) in enumerate(pieces):
        arr[i].src, arr[i].dst, arr[i].bytes = src.ctypes.data + off, dst_orc.ctypes.data + off, ln
    oracle.oracle_slab_move(arr, len(pieces))
    assert np.array_equal(dst_eng, dst_orc)


def test_copy_slabs_rejects_misaligned(engine):
    from nvshare_b200.engine import EngineError
    buf = np.zeros(4096, dtype=np.uint8)
    with pytest.raises(EngineError):
        engine.copy_slabs([(buf.ctypes.data + 8, buf.ctypes.data + 1024, 64)], variant="tma")
    with pytest.raises(EngineError):
        engine.copy_slabs([(buf.ctypes.data, buf.ctypes.data + 1024, 24)], variant="tma")
    assert engine.copy_slabs([], variant="tma") >= 0         # empty list is fine


def test_partial_eviction_takes_least_recently_fetched_first(engine):
    a = engine.alloc(16 * MiB)
    engine.fetch_all()                      # epoch 1: a
    b = engine.alloc(16 * MiB)              # resident mode: mapped at once, same epoch as a's
    engine.evict(0)
    engine.fetch_all()                      # epoch 2: a and b
    c = engine.alloc(16 * MiB)
    st0 = engine.stats()
    assert st0["resident_bytes"] == 48 * MiB
    rep = engine.evict(10 * MiB)            # needs two 8 MiB chunks; a's and b's are tied, lowest VA first
    assert rep["bytes"] == 16 * MiB
    st = engine.stats()
    assert st["resident_bytes"] == 32 * MiB and st["swapped_bytes"] == 16 * MiB
    rep = engine.fetch_all()
    assert rep["bytes"] == 16 * MiB         # only what was out comes back
    for p in (a, b, c):
        engine.free(p)


def test_free_while_swapped_returns_backing(engine):
    p = engine.alloc(24 * MiB)
    engine.fetch_all()
    engine.pattern_fill(p, 24 * MiB // 8)
    engine.evict(0)
    used = engine.stats()["host_pool_used"]
    assert used == 24 * MiB
    engine.free(p)
    st = engine.stats()
    assert st["host_pool_used"] == 0 and st["swapped_bytes"] == 0 and st["n_allocs"] == 0
    q = engine.alloc(24 * MiB)              # pool is reused, not grown
    engine.fetch_all(); engine.evict(0)
    assert engine.stats()["host_pool_bytes"] == 64 * MiB
    engine.free(q)


def test_small_allocations_pass_through(engine, fake):
    base = fake.fake_cuda_phys_used()
    p = engine.alloc(1000)
    st = engine.stats()
    assert st["passthrough_bytes"] == 1000 and st["va_bytes"] == 0
    assert fake.fake_cuda_phys_used() == base + 1000        # plain device memory, resident for life
    engine.evict(0)
    view(p, 1000)[:] = 7                                    # still accessible
    engine.free(p)


def test_free_of_foreign_pointer(engine):
    from nvshare_b200.engine import EngineError
    with pytest.raises(EngineError) as ei:
        engine.free(0x1000)
    assert ei.value.rc == -2                                # NVS_E_NOT_OURS: the hook falls through to cuMemFree


def test_alloc_zero_is_invalid_value(engine):
    from nvshare_b200.engine import EngineError
    with pytest.raises(EngineError) as ei:
        engine.alloc(0)
    assert ei.value.rc == 1                                 # CUDA_ERROR_INVALID_VALUE


def test_fetch_times_out_when_hbm_never_frees(fake, tmp_path):
    from nvshare_b200 import engine as E
    ledger = tmp_path / "ledger"
    code = textwrap.dedent(f"""
        import ctypes as C, sys
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        e = E.Engine(chunk_bytes=8 << 20, host_arena_bytes=64 << 20, oom_wait_ms=200)
        p = e.alloc(64 << 20)
        try:
            e.fetch_all()
            print("UNEXPECTED")
        except E.EngineError as ex:
            print("RC", ex.rc)
    """)
    env = dict(__import__("os").environ, FAKE_CUDA_TOTAL_MIB="32", FAKE_CUDA_LEDGER=str(ledger))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=60)
    assert "RC -6" in r.stdout, r.stdout + r.stderr         # NVS_E_TIMEOUT


def test_resident_allocation_that_cannot_get_hbm_fails_clean(fake, tmp_path):
    """The lock holder asks for more than the GPU can give (cuMemAlloc -> nvs_alloc in resident mode): the call
    fails with CUDA_ERROR_OUT_OF_MEMORY after the wait, what it had mapped so far goes back, the counters return
    to where they were, and the engine goes on working."""
    ledger = tmp_path / "ledger"
    code = textwrap.dedent(f"""
        import ctypes as C, sys
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.fake_cuda_phys_used.restype = C.c_uint64
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        MiB = 1 << 20
        e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, oom_wait_ms=200, prepin=0, shared_pool_path=None)
        e.set_resident_mode(True)
        keep = e.alloc(24 * MiB)                       # resident at once: the holder's allocations are usable immediately
        before = e.stats()
        used = fake.fake_cuda_phys_used()
        try:
            e.alloc(64 * MiB); print("UNEXPECTED")
        except E.EngineError as ex:
            print("RC", ex.rc)
        after = e.stats()
        print("SAME", all(after[k] == before[k] for k in ("resident_bytes", "unbacked_bytes", "swapped_bytes", "va_bytes")))
        print("PHYS", fake.fake_cuda_phys_used() == used)
        e.pattern_fill(keep, 24 * MiB // 8, seed=5); e.evict(0); e.fetch_all()
        print("BAD", e.pattern_verify(keep, 24 * MiB // 8, seed=5))
        small = e.alloc(16 * MiB); print("LATER", e.stats()["resident_bytes"] // MiB)
    """)
    env = dict(__import__("os").environ, FAKE_CUDA_TOTAL_MIB="64", FAKE_CUDA_LEDGER=str(ledger))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=60)
    assert "RC 2" in r.stdout and "UNEXPECTED" not in r.stdout, r.stdout + r.stderr       # CUDA_ERROR_OUT_OF_MEMORY
    assert "SAME True" in r.stdout and "PHYS True" in r.stdout and "BAD 0" in r.stdout and "LATER 40" in r.stdout, r.stdout + r.stderr


def test_timed_out_fetch_leaves_a_consistent_table(fake, tmp_path):
    """A fetch that gives up half-way must not mark a chunk resident before its
    data is back: after the HBM hog goes away a second fetch restores everything."""
    ledger = tmp_path / "ledger"
    code = textwrap.dedent(f"""
        import ctypes as C, sys
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        MiB = 1 << 20
        e = E.Engine(chunk_bytes=8 * MiB, batch_bytes=32 * MiB, burst_bytes=8 * MiB, host_arena_bytes=64 * MiB,
                     oom_wait_ms=300, elide_constant=0, shared_pool_path=None)
        p = e.alloc(24 * MiB); e.fetch_all()
        e.pattern_fill(p, 24 * MiB // 8, first_index=3, seed=99)
        e.evict(0)
        hog = C.c_uint64()
        assert fake.cuMemAlloc_v2(C.byref(hog), C.c_size_t(20 * MiB)) == 0
        try:
            e.fetch_all(); print("UNEXPECTED")
        except E.EngineError as ex:
            print("RC", ex.rc)
        st = e.stats()
        print("RESIDENT", st["resident_bytes"] // MiB, "SWAPPED", st["swapped_bytes"] // MiB)
        assert fake.cuMemFree_v2(hog) == 0
        e.fetch_all()
        print("BAD", e.pattern_verify(p, 24 * MiB // 8, first_index=3, seed=99))
        st = e.stats()
        print("POOL_USED", st["host_pool_used"] - st["retained_bytes"])    # kept copies are reclaimable, not in use
    """)
    env = dict(__import__("os").environ, FAKE_CUDA_TOTAL_MIB="40", FAKE_CUDA_LEDGER=str(ledger))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=60)
    out = r.stdout
    assert "RC -6" in out and "UNEXPECTED" not in out, out + r.stderr
    assert "SWAPPED 0" not in out, out                      # something was still out when it gave up
    assert "BAD 0" in out and "POOL_USED 0" in out, out + r.stderr


def test_evicted_memory_is_unmapped(artefacts):
    """An access to an evicted slab must fault (fake driver: SIGSEGV), i.e. the
    physical memory really went away."""
    code = textwrap.dedent(f"""
        import ctypes as C, sys
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        e = E.Engine(chunk_bytes=8 << 20, host_arena_bytes=64 << 20)
        p = e.alloc(16 << 20); e.fetch_all()
        C.memset(p, 1, 16 << 20); print("resident ok", flush=True)
        e.evict(0)
        C.memset(p, 1, 4096); print("STILL MAPPED", flush=True)
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=60)
    assert "resident ok" in r.stdout and "STILL MAPPED" not in r.stdout
    assert r.returncode == -11


def test_peer_tier_is_preferred_and_striped(fake):
    from nvshare_b200 import engine as E
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=32 * MiB, peers=[1, 2], peer_capacity_bytes=32 * MiB,
                 prepin=0, elide_constant=0)
    try:
        p = e.alloc(80 * MiB)
        e.fetch_all()
        e.pattern_fill(p, 80 * MiB // 8, seed=5)
        rep = e.evict(0)
        # two peers x 32 MiB capacity take 64 MiB, the remaining 16 MiB spill to pinned host memory
        assert rep["peer_bytes"] == 64 * MiB and rep["host_bytes"] == 16 * MiB
        st = e.stats()
        assert st["peer_pool_used"] == 64 * MiB and st["host_pool_used"] == 16 * MiB
        rep = e.fetch_all()
        assert rep["peer_bytes"] == 64 * MiB and rep["host_bytes"] == 16 * MiB
        assert e.pattern_verify(p, 80 * MiB // 8, seed=5) == 0
        e.free(p)
    finally:
        e.close()


def test_same_filled_slabs_are_not_moved(fake, oracle):
    """Slabs whose 64-bit words are all equal are described, not copied: zero
    pages, ones() tensors (the reference's own test data), memset workspaces."""
    from nvshare_b200 import engine as E
    # (background pre-cleaning off: it may copy a chunk before the test has written it, and then the byte counts
    # below depend on timing; tests/test_policy_fake.py and tests/test_retention_fake.py cover it)
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, batch_bytes=24 * MiB, preclean=0)
    try:
        assert e.cfg.elide_constant == 1
        p = e.alloc(40 * MiB)                                # 20 slabs in 5 chunks
        e.fetch_all()
        ones = np.float32(1.0).view(np.uint32)
        v = view(p, 40 * MiB).view(np.uint32)
        v[:] = ones                                          # everything same-filled ...
        v[(6 * MiB) // 4 + 17] = 0                           # ... except one word in slab 3
        e.pattern_fill(p + 16 * MiB, (4 * MiB) // 8, seed=11)  # ... and slabs 8, 9 (position-dependent)
        rep = e.evict(0)
        assert rep["bytes"] == 3 * SLAB and rep["elided_bytes"] == 17 * SLAB
        st = e.stats()
        assert st["swapped_bytes"] == 40 * MiB
        assert st["host_pool_used"] == 2 * 8 * MiB           # only the 2 chunks with a real slab keep backing
        rep = e.fetch_all()
        assert rep["bytes"] == 3 * SLAB and rep["elided_bytes"] == 17 * SLAB
        got = view(p, 40 * MiB).view(np.uint32)
        want = np.full(40 * MiB // 4, ones, dtype=np.uint32)
        want[(6 * MiB) // 4 + 17] = 0
        tmp = np.empty(4 * MiB // 8, dtype=np.uint64)
        oracle.oracle_pattern_fill(tmp.ctypes.data, tmp.size, 0, 11)
        want[(16 * MiB) // 4:(20 * MiB) // 4] = tmp.view(np.uint32)
        assert np.array_equal(got, want)
        # a second cycle after the application changed a formerly same-filled slab
        view(p, 16)[:] = 9
        rep = e.evict(0)
        # slab 0 is no longer same-filled and has to go out; slabs 3, 8 and 9 still match the backing
        # copies kept from the first cycle (clean-slab skip) and are not copied again
        assert rep["bytes"] == 1 * SLAB and rep["elided_bytes"] == 16 * SLAB and rep["clean_bytes"] == 3 * SLAB
        e.fetch_all()
        want.view(np.uint8)[:16] = 9
        assert np.array_equal(view(p, 40 * MiB).view(np.uint32), want)
        e.free(p)
    finally:
        e.close()


def test_bad_geometry_is_rejected(fake):
    from nvshare_b200 import engine as E
    with pytest.raises(E.EngineError):
        E.Engine(chunk_bytes=3 * MiB)                       # not a multiple of the 2 MiB slab
    with pytest.raises(E.EngineError):
        E.Engine(tma_stages=1)
    with pytest.raises(E.EngineError):
        E.Engine(tma_warps=4, tma_stages=6, tma_tile_bytes=32768)   # 768 KiB of shared memory


def test_stats_file(fake, tmp_path):
    import json
    from nvshare_b200 import engine as E
    path = tmp_path / "stats.jsonl"
    # (background pre-cleaning off: a chunk it had written back between the fetch and the eviction would be found
    # clean and not be counted in "bytes" -- once in some fifteen runs of the suite)
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, stats_path=str(path), elide_constant=0, preclean=0)
    p = e.alloc(16 * MiB); e.fetch_all(); e.evict(0); e.fetch_all(); e.free(p); e.close()
    recs = [json.loads(l) for l in path.read_text().splitlines()]
    assert [r["op"] for r in recs] == ["fetch", "evict", "fetch"]
    assert recs[1]["bytes"] == 16 * MiB and recs[1]["slabs"] == 8 and recs[1]["launches"] >= 1


# ---- nvs_host_io: copies between host memory and a range that is not on the GPU (SURVEY 8f rank 3)

def test_host_io_return_codes(fake):
    from nvshare_b200 import engine as E
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, oom_wait_ms=300, prepin=0)
    try:
        buf = np.arange(4096, dtype=np.uint8)
        p = e.alloc(20 * MiB)
        assert e.host_io(p, buf.ctypes.data, 4096, False) == -9          # never written: nothing to read back
        e.fetch_all()
        assert e.host_io(p, buf.ctypes.data, 4096, True) == -9           # resident: the device path must be used
        assert e.host_io(p + 20 * MiB + 2 * MiB - 8, buf.ctypes.data, 16, True) == -2   # runs off the allocation's end
        assert e.host_io(0x1000, buf.ctypes.data, 16, True) == -2        # not ours
        small = e.alloc(4096)                                            # passthrough allocation: plain device memory
        assert e.host_io(small, buf.ctypes.data, 16, True) == -2
        e.evict(0)
        assert e.host_io(p, buf.ctypes.data, 4096, True) == 0
        assert e.stats()["host_io_bytes_total"] == 4096
    finally:
        e.close()


def test_host_io_load_before_first_residency_reads_zero_elsewhere(fake):
    """Uploading into a fresh allocation without the GPU: the bytes written arrive,
    everything else in the chunk reads 0 (never another client's stale pool pages)."""
    from nvshare_b200 import engine as E
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, oom_wait_ms=300, prepin=0)
    try:
        # dirty the pool first: whatever backs the next allocation has non-zero bytes in it
        q = e.alloc(24 * MiB); e.fetch_all(); view(q, 24 * MiB)[:] = 0xAB; e.evict(0); e.fetch_all(); e.free(q)
        e.evict(0)
        p = e.alloc(24 * MiB)
        src = np.random.default_rng(1).integers(1, 256, 9 * MiB + 13, dtype=np.uint8)
        lo = 3 * MiB + 5                                                  # spans chunks 0 and 1, ragged at both ends
        assert e.host_io(p + lo, src.ctypes.data, len(src), True) == 0
        st = e.stats()
        assert st["swapped_bytes"] == 16 * MiB and st["unbacked_bytes"] == 8 * MiB and st["resident_bytes"] == 0
        back = np.empty(len(src) + 64, dtype=np.uint8)
        assert e.host_io(p + lo - 32, back.ctypes.data, len(back), False) == 0     # readable again without the GPU
        assert not back[:32].any() and np.array_equal(back[32:32 + len(src)], src) and not back[32 + len(src):].any()
        rep = e.fetch_all()
        got = view(p, 24 * MiB)
        assert np.array_equal(got[lo:lo + len(src)], src)
        assert not got[:lo].any() and not got[lo + len(src):].any()
        assert rep["bytes"] == 12 * MiB                                   # only the six slabs that were touched moved
    finally:
        e.close()


def test_host_io_large_copies_are_split_over_threads(fake):
    """A run of 32 MiB or more inside one chunk is copied by several threads (par_memcpy): with the production chunk
    size (256 MiB) that is every model-sized upload.  Ragged ends, both directions, then the device's view."""
    from nvshare_b200 import engine as E
    e = E.Engine(chunk_bytes=128 * MiB, host_arena_bytes=128 * MiB, oom_wait_ms=300, prepin=0, elide_constant=0, retain=0)
    try:
        p = e.alloc(128 * MiB)
        src = np.random.default_rng(7).integers(0, 256, 101 * MiB + 4099, dtype=np.uint8)
        lo = 5 * MiB + 17
        assert e.host_io(p + lo, src.ctypes.data, len(src), True) == 0
        back = np.empty(len(src), dtype=np.uint8)
        assert e.host_io(p + lo, back.ctypes.data, len(back), False) == 0
        assert np.array_equal(back, src)
        e.fetch_all()
        got = view(p, 128 * MiB)
        assert np.array_equal(got[lo:lo + len(src)], src) and not got[:lo].any() and not got[lo + len(src):].any()
    finally:
        e.close()


def test_host_io_on_same_filled_slabs(fake):
    from nvshare_b200 import engine as E
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, oom_wait_ms=300, prepin=0, elide_constant=1)
    try:
        p = e.alloc(16 * MiB); e.fetch_all()
        words = np.ctypeslib.as_array((C.c_uint64 * (16 * MiB // 8)).from_address(p))
        words[:] = 0x0102030405060708                                     # every slab same-filled ...
        view(p, 16 * MiB)[5 * MiB] ^= 0xFF                                # ... but slab 2
        rep = e.evict(0)
        assert rep["bytes"] == 2 * MiB and rep["elided_bytes"] == 14 * MiB
        expect = np.frombuffer(np.full(16 * MiB // 8, 0x0102030405060708, dtype=np.uint64).tobytes(), dtype=np.uint8).copy()
        expect[5 * MiB] ^= 0xFF
        back = np.empty(6 * MiB + 3, dtype=np.uint8)
        assert e.host_io(p + 1 * MiB + 1, back.ctypes.data, len(back), False) == 0   # unaligned read across const + real slabs
        assert np.array_equal(back, expect[1 * MiB + 1:1 * MiB + 1 + len(back)])
        patch = np.arange(100, dtype=np.uint8)
        assert e.host_io(p + 9 * MiB + 3, patch.ctypes.data, 100, True) == 0         # into a same-filled slab of chunk 1
        expect[9 * MiB + 3:9 * MiB + 103] = patch
        e.fetch_all()
        assert np.array_equal(view(p, 16 * MiB), expect)
    finally:
        e.close()


def test_best_effort_eviction_never_waits_for_backing_space(fake, tmp_path):
    """nvs_evict_best_effort (used for evictions done as a favour under memory pressure):
    with the backing pool full it moves what fits, returns 0 at once and leaves the rest
    resident and intact; the ordinary nvs_evict waits, then overflows into a private arena."""
    import time
    from nvshare_b200 import engine as E
    pool = tmp_path / "pool"
    e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, batch_bytes=16 * MiB, shared_pool_path=str(pool),
                 shared_pool_bytes=64 * MiB, oom_wait_ms=10000, elide_constant=0, prepin=0, retain=0)
    try:
        p = e.alloc(96 * MiB); e.fetch_all()
        e.pattern_fill(p, 96 * MiB // 8, seed=21)
        t0 = time.time()
        rep = e.evict_best_effort(0)
        assert time.time() - t0 < 1.5
        st = e.stats()
        assert rep["bytes"] == 64 * MiB == st["swapped_bytes"] and st["resident_bytes"] == 32 * MiB
        assert st["host_pool_used"] == 64 * MiB
        # the blocking flavour waits for units; nobody returns any, so after the grace period it pins
        # a private overflow arena beside the shared pool and completes
        t0 = time.time()
        rep = e.evict(0)
        st = e.stats()
        assert time.time() - t0 >= 1.9 and rep["bytes"] == 32 * MiB and st["resident_bytes"] == 0
        assert st["host_pool_bytes"] == 128 * MiB and st["host_pool_used"] == 96 * MiB
        e.fetch_all()
        assert e.pattern_verify(p, 96 * MiB // 8, seed=21) == 0
        assert e.stats()["host_pool_used"] == 0
        rep = e.evict_best_effort(16 * MiB)                  # partial request, plenty of room: behaves like nvs_evict
        assert rep["bytes"] == 16 * MiB
        e.fetch_all()
        assert e.pattern_verify(p, 96 * MiB // 8, seed=21) == 0
        e.free(p)
    finally:
        e.close()


def test_allocation_by_the_lock_holder_stops_waiting_when_the_lock_goes(fake, tmp_path):
    """Seen with a ResNet-50 client: the quantum ended while the holder's cuMemAlloc was waiting for HBM the other client still
    had; the allocation kept the engine's entry lock for oom_wait_ms (120 s), the hand-off's eviction queued
    behind it, and the daemon rightly ignored pressure from a client that no longer held the lock.  Now the
    wait ends with the lock: what is mapped stays, the rest is virtual until the next fetch."""
    ledger = tmp_path / "ledger"
    code = textwrap.dedent(f"""
        import ctypes as C, sys, threading, time
        sys.path.insert(0, {str(ROOT)!r})
        fake = C.CDLL({str(FAKE_DIR / 'libcuda.so.1')!r}, mode=C.RTLD_GLOBAL)
        fake.cuInit(0); ctx = C.c_void_p(); fake.cuDevicePrimaryCtxRetain(C.byref(ctx), 0); fake.cuCtxSetCurrent(ctx)
        from nvshare_b200 import engine as E
        MiB = 1 << 20
        e = E.Engine(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, oom_wait_ms=60000, prepin=0, preclean=0)
        hog = C.c_uint64()
        assert fake.cuMemAlloc_v2(C.byref(hog), C.c_size_t(40 * MiB)) == 0      # "the other client": 40 of 64 MiB
        e.set_resident_mode(True)                                              # we hold the lock
        out = {{}}
        def alloc():
            fake.cuCtxSetCurrent(ctx)
            t0 = time.time(); out["p"] = e.alloc(48 * MiB); out["s"] = time.time() - t0
        th = threading.Thread(target=alloc); th.start()
        time.sleep(0.5)
        assert th.is_alive()                                                   # waiting for HBM
        t0 = time.time()
        e.set_resident_mode(False)                                             # DROP_LOCK: the quantum is over
        th.join(10)
        assert not th.is_alive() and time.time() - t0 < 2.0, "the allocation kept waiting without the lock"
        st = e.stats()
        print("RESIDENT", st["resident_bytes"] // MiB, "UNBACKED", st["unbacked_bytes"] // MiB, flush=True)
        t0 = time.time(); e.evict(0); print("EVICT_S %.2f" % (time.time() - t0), flush=True)   # the hand-off's eviction is not stuck
        assert fake.cuMemFree_v2(hog) == 0
        e.fetch_all(); e.pattern_fill(out["p"], 48 * MiB // 8, seed=1)
        print("BAD", e.pattern_verify(out["p"], 48 * MiB // 8, seed=1), flush=True)
        e.free(out["p"]); e.close()
    """)
    env = dict(__import__("os").environ, FAKE_CUDA_TOTAL_MIB="64", FAKE_CUDA_LEDGER=str(ledger))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "BAD 0" in r.stdout, r.stdout + r.stderr
    res, unb = (int(x) for x in r.stdout.split("RESIDENT")[1].split()[0:3:2])
    assert res + unb == 48 and 0 < res <= 24 and unb >= 24, r.stdout          # part mapped, the rest virtual
    assert float(r.stdout.split("EVICT_S")[1].split()[0]) < 2.0
