"""Parity tests proper: the sm_90a kernels and the swap engine on a real H100,
called through the C-ABI (libnvs_engine.so), checked bit-exact against the CPU
oracle (oracle/nvshare_oracle.c) on the same seeded inputs, plus
size-independent round-trip properties at sizes the oracle would take too long
for.  torch is used only to obtain a CUDA context and raw device / pinned
buffers."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from nvs_testlib import ORACLE

pytestmark = pytest.mark.gpu

MiB = 1 << 20
GiB = 1 << 30
SLAB = 2 * MiB


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("these tests need a GPU")
    torch.cuda.init()
    torch.zeros(1, device="cuda")          # makes the primary context current on this thread
    return torch


@pytest.fixture(scope="module")
def oracle(artefacts):
    lib = C.CDLL(str(ORACLE / "liboracle.so"))
    lib.oracle_pattern_mismatches.restype = C.c_uint64
    lib.oracle_pattern_mismatches.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    lib.oracle_pattern_fill.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    lib.oracle_slab_move.argtypes = [C.c_void_p, C.c_uint32]
    return lib


@pytest.fixture()
def engine(torch_cuda, artefacts):
    from nvshare_b200 import engine as E
    # production defaults (256 MiB chunks, host tier on the copy engines, clean-slab skip) except background
    # pre-cleaning: it would write chunks back while a test is still filling them and make the byte counts
    # asserted below depend on timing (it has its own test)
    e = E.Engine(preclean=0)
    yield e
    e.close()


def ragged_pieces(rng, size, n):
    cuts = sorted(set([0, size] + [int(x) & ~15 for x in rng.integers(16, size - 16, n - 1)]))
    pieces = [(cuts[i], cuts[i + 1] - cuts[i]) for i in range(len(cuts) - 1)]
    out = []
    for off, ln in pieces:                  # a descriptor never exceeds one slab
        while ln > 0:
            step = min(ln, SLAB)
            out.append((off, step))
            off += step
            ln -= step
    rng.shuffle(out)
    return out


@pytest.mark.parametrize("variant,grid", [("tma", 1), ("tma", 8), ("tma", 132), ("ldg", 8), ("ldg", 132), ("ce", 0)])
def test_copy_kernels_match_oracle_device_to_device(torch_cuda, engine, oracle, variant, grid):
    torch = torch_cuda
    g = torch.Generator(device="cpu").manual_seed(1234)
    size = 24 * MiB
    src_h = torch.randint(0, 256, (size,), dtype=torch.uint8, generator=g)
    src = src_h.cuda()
    dst = torch.zeros(size, dtype=torch.uint8, device="cuda")
    pieces = ragged_pieces(np.random.default_rng(5), size, 40)
    ms = engine.copy_slabs([(src.data_ptr() + o, dst.data_ptr() + o, n) for o, n in pieces], variant=variant, grid=grid)
    assert ms > 0
    # oracle: the same descriptor list applied with memcpy on host copies
    from nvshare_b200.engine import CopyDesc
    src_np = src_h.numpy()
    want = np.zeros(size, dtype=np.uint8)
    arr = (CopyDesc * len(pieces))()
    for i, (o, n) in enumerate(pieces):
        arr[i].src, arr[i].dst, arr[i].bytes = src_np.ctypes.data + o, want.ctypes.data + o, n
    oracle.oracle_slab_move(arr, len(pieces))
    torch.cuda.synchronize()
    assert np.array_equal(dst.cpu().numpy(), want)


@pytest.mark.parametrize("variant", ["tma", "ldg", "ce"])
def test_copy_kernels_to_and_from_pinned_host(torch_cuda, engine, oracle, variant):
    """The swap path itself: HBM -> pinned host -> HBM, each leg checked against the oracle."""
    torch = torch_cuda
    size = 64 * MiB
    words = size // 8
    dev = torch.empty(size, dtype=torch.uint8, device="cuda")
    host = torch.zeros(size, dtype=torch.uint8).pin_memory()
    back = torch.zeros(size, dtype=torch.uint8, device="cuda")
    engine.pattern_fill(dev.data_ptr(), words, first_index=99, seed=3)
    slabs = [(i * SLAB, SLAB) for i in range(size // SLAB)]
    engine.copy_slabs([(dev.data_ptr() + o, host.data_ptr() + o, n) for o, n in slabs], variant=variant, grid=8)
    assert oracle.oracle_pattern_mismatches(host.data_ptr(), words, 99, 3) == 0      # CPU reads what the GPU wrote
    engine.copy_slabs([(host.data_ptr() + o, back.data_ptr() + o, n) for o, n in reversed(slabs)], variant=variant,
                      grid=8)
    assert engine.pattern_verify(back.data_ptr(), words, first_index=99, seed=3) == 0
    assert torch.equal(dev, back)


def test_pattern_kernels_agree_with_oracle(torch_cuda, engine, oracle):
    torch = torch_cuda
    words = (8 * MiB) // 8
    dev = torch.empty(words, dtype=torch.int64, device="cuda")
    engine.pattern_fill(dev.data_ptr(), words, first_index=1 << 40, seed=77)
    host = dev.cpu().numpy()
    assert oracle.oracle_pattern_mismatches(host.ctypes.data, words, 1 << 40, 77) == 0
    want = np.empty(words, dtype=np.uint64)
    oracle.oracle_pattern_fill(want.ctypes.data, words, 1 << 40, 77)
    assert np.array_equal(host.view(np.uint64), want)
    dev[12345] ^= 1                                                                   # one flipped bit is seen
    assert engine.pattern_verify(dev.data_ptr(), words, first_index=1 << 40, seed=77) == 1


def test_edge_cases(torch_cuda, engine):
    torch = torch_cuda
    buf = torch.zeros(4 * MiB, dtype=torch.uint8, device="cuda")
    out = torch.zeros(4 * MiB, dtype=torch.uint8, device="cuda")
    buf[:] = torch.arange(4 * MiB, device="cuda") % 251
    p, q = buf.data_ptr(), out.data_ptr()
    assert engine.copy_slabs([], variant="tma") >= 0                                  # empty
    engine.copy_slabs([(p, q, 16)], variant="tma", grid=4)                            # minimum bulk size
    engine.copy_slabs([(p + 16, q + 16, 0), (p + 32, q + 32, 48)], variant="tma")     # zero-length descriptor skipped
    engine.copy_slabs([(p + 1024, q + 1024, 1000)], variant="ldg")                    # 8-byte tail on the LDG variant
    torch.cuda.synchronize()
    assert torch.equal(out[:16], buf[:16]) and torch.equal(out[32:80], buf[32:80])
    assert int(out[16:32].sum()) == 0
    assert torch.equal(out[1024:2024], buf[1024:2024]) and int(out[2024:2048].sum()) == 0
    # many tiny descriptors (more descriptors than CTAs x stages)
    n = 4096
    descs = [(p + 4096 + i * 256, q + 4096 + i * 256, 256) for i in range(n)]
    engine.copy_slabs(descs, variant="tma", grid=16)
    torch.cuda.synchronize()
    assert torch.equal(out[4096:4096 + n * 256], buf[4096:4096 + n * 256])


def test_engine_round_trips_release_hbm(torch_cuda, engine):
    torch = torch_cuda
    sizes = [3 * GiB + 6 * MiB, 512 * MiB, 2 * MiB, 70 * MiB]
    ptrs = [engine.alloc(s) for s in sizes]
    engine.fetch_all()
    for k, (p, s) in enumerate(zip(ptrs, sizes)):
        engine.pattern_fill(p, s // 8, first_index=k << 36, seed=42)
    total = sum((s + SLAB - 1) // SLAB * SLAB for s in sizes)
    free_resident, _ = torch.cuda.mem_get_info()
    for cycle in range(2):
        rep = engine.evict(0)
        # the first time everything crosses the link; the second time nothing has changed since the
        # backing copies were written, the hash scan finds every slab clean and nothing is copied
        assert rep["bytes"] + rep["clean_bytes"] == total and rep["bytes"] == (total if cycle == 0 else 0)
        assert rep["slabs"] == rep["bytes"] // SLAB
        free_out, _ = torch.cuda.mem_get_info()
        assert free_out - free_resident >= total - 256 * MiB                          # the HBM really went back
        assert engine.stats()["resident_bytes"] == 0
        rep = engine.fetch_all()
        assert rep["bytes"] == total
        for k, (p, s) in enumerate(zip(ptrs, sizes)):
            assert engine.pattern_verify(p, s // 8, first_index=k << 36, seed=42) == 0
    # partial eviction, then the application "computes" on everything again
    rep = engine.evict(1 * GiB)
    assert 1 * GiB <= rep["bytes"] + rep["clean_bytes"] <= 1 * GiB + 256 * MiB
    engine.fetch_all()
    assert engine.pattern_verify(ptrs[0], sizes[0] // 8, first_index=0, seed=42) == 0
    st = engine.stats()
    assert st["kernel_launches_total"] > 0
    for p in ptrs:
        engine.free(p)


@pytest.mark.parametrize("evict_v,fetch_v", [("ldg", "ldg"), ("ce", "ce"), ("tma", "tma")])
def test_engine_variants(torch_cuda, artefacts, evict_v, fetch_v):
    from nvshare_b200 import engine as E
    e = E.Engine(evict_variant=evict_v, fetch_variant=fetch_v)
    try:
        p = e.alloc(1 * GiB + 2 * MiB)
        e.fetch_all()
        e.pattern_fill(p, (1 * GiB + 2 * MiB) // 8, seed=9)
        e.evict(0)
        e.fetch_all()
        assert e.pattern_verify(p, (1 * GiB + 2 * MiB) // 8, seed=9) == 0
    finally:
        e.close()


def test_same_filled_slabs_are_elided_and_recreated(torch_cuda, engine, oracle):
    """nvs_slab_scan / nvs_slab_splat on the GPU against the oracle's per-slab test."""
    torch = torch_cuda
    size = 1 * GiB + 4 * MiB
    n = size // 4
    p = engine.alloc(size)
    engine.fetch_all()

    class Raw:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}

    t = torch.as_tensor(Raw(p, n), device="cuda")
    t.fill_(1.0)                                             # the reference workload's data: torch.ones
    g = torch.Generator(device="cpu").manual_seed(3)
    noisy_slabs = sorted(set(torch.randint(0, size // SLAB, (37,), generator=g).tolist()))
    for sidx in noisy_slabs:                                 # one differing word somewhere in 37 slabs
        t[sidx * (SLAB // 4) + (sidx * 7919) % (SLAB // 4)] = 3.0
    torch.cuda.synchronize()
    host = t.cpu().numpy()
    oracle.oracle_slab_is_const.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    val = C.c_uint64()
    want_const = sum(oracle.oracle_slab_is_const(host.ctypes.data + i * SLAB, SLAB, C.byref(val))
                     for i in range(size // SLAB))
    assert want_const == size // SLAB - len(noisy_slabs)
    rep = engine.evict(0)
    assert rep["elided_bytes"] == want_const * SLAB and rep["bytes"] == len(noisy_slabs) * SLAB
    rep = engine.fetch_all()
    assert rep["elided_bytes"] == want_const * SLAB and rep["bytes"] == len(noisy_slabs) * SLAB
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), host)             # bit-exact, splatted and copied slabs alike
    del t
    engine.free(p)


def test_scan_hash_kernel_matches_the_oracle(torch_cuda, engine, oracle):
    """nvs_slab_scan's 128-bit content hash on the GPU against oracle_slab_hash (plain C) on the same
    bytes, bit for bit: whole slabs, a ragged one, a same-filled one; one flipped bit changes it."""
    torch = torch_cuda
    from nvshare_b200 import engine as E
    oracle.oracle_slab_hash.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64 * 2)]
    n_slabs = 24
    buf = torch.empty(n_slabs * SLAB, dtype=torch.uint8, device="cuda")
    buf.random_(0, 256, generator=torch.Generator(device="cuda").manual_seed(17))
    buf[5 * SLAB:6 * SLAB] = 0x3C                            # a same-filled slab
    torch.cuda.synchronize()
    base = buf.data_ptr()
    descs = [(base + i * SLAB, 0, SLAB) for i in range(n_slabs - 1)] + [(base + (n_slabs - 1) * SLAB, 0, 333 * 16)]
    out = E.scan_slabs(engine, descs, want_hash=True)
    host = buf.cpu().numpy()
    for i, ((src, _, nb), o) in enumerate(zip(descs, out)):
        want = (C.c_uint64 * 2)()
        oracle.oracle_slab_hash(host.ctypes.data + (src - base), nb, C.byref(want))
        assert (o["h0"], o["h1"]) == (want[0], want[1]), f"slab {i}"
        assert o["is_const"] == (1 if i == 5 else 0)
    assert len({(o["h0"], o["h1"]) for o in out}) == n_slabs                # position-dependent: all different
    buf[7 * SLAB + 1234567] ^= 0x20
    torch.cuda.synchronize()
    again = E.scan_slabs(engine, descs[7:8], want_hash=True)[0]
    assert (again["h0"], again["h1"]) != (out[7]["h0"], out[7]["h1"])
    quick = E.scan_slabs(engine, descs, want_hash=False)
    assert all(q["h0"] == 0 and q["h1"] == 0 for q in quick) and [q["is_const"] for q in quick] == [o["is_const"] for o in out]


def test_clean_slabs_are_not_copied_again_and_one_changed_word_is(torch_cuda, engine):
    """VERDICT #3 on the GPU: what has not changed since its backing copy was written does not cross the
    link again; a single word changed in a "clean" slab is seen after the round trip."""
    torch = torch_cuda
    size = 2 * GiB + 6 * MiB
    p = engine.alloc(size)
    engine.fetch_all()
    engine.pattern_fill(p, size // 8, first_index=11, seed=5)
    total = (size + SLAB - 1) // SLAB * SLAB
    r = engine.evict(0)
    assert r["bytes"] == total and r["clean_bytes"] == 0
    engine.fetch_all()
    assert engine.stats()["retained_bytes"] == total
    r = engine.evict(0)
    assert r["bytes"] == 0 and r["clean_bytes"] == total and r["ce_calls"] == 0 and r["scanned_bytes"] == total
    engine.fetch_all()

    class Raw:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}

    t = torch.as_tensor(Raw(p, size // 8), device="cuda")
    word = 517 * (SLAB // 8) + 4242                          # slab 517: in the third chunk
    t[word] += 1
    torch.cuda.synchronize()
    expect = t.cpu()
    r = engine.evict(0)
    assert r["bytes"] == SLAB and r["clean_bytes"] == total - SLAB
    engine.fetch_all()
    torch.cuda.synchronize()
    assert torch.equal(t.cpu(), expect)
    assert engine.pattern_verify(p, word, first_index=11, seed=5) == 0       # everything before it still the pattern
    del t
    engine.free(p)


def test_background_precleaning_with_the_fused_copy_hash_kernel(torch_cuda, artefacts):
    """nvs_slab_scan with a destination (copy + hash in one pass) on the GPU: while the "owner" holds the lock and a
    kernel keeps rewriting one allocation, the pre-cleaner writes everything back; the eviction then copies only
    what the recorded hashes do not vouch for, and every byte survives the round trip."""
    import time
    torch = torch_cuda
    from nvshare_b200 import engine as E
    with E.Engine() as e:
        size = 1 * GiB
        quiet, busy = e.alloc(size), e.alloc(size)
        e.fetch_all()
        e.pattern_fill(quiet, size // 8, first_index=3, seed=8)

        class Raw:
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}

        t = torch.as_tensor(Raw(busy, size // 8), device="cuda")
        t.copy_(torch.arange(size // 8, device="cuda", dtype=torch.int64))      # position-dependent: nothing same-filled
        e.set_resident_mode(True)
        deadline = time.time() + 20
        while e.stats()["precleaned_bytes_total"] < 2 * size and time.time() < deadline:
            t.add_(1)                                        # the application keeps writing while its memory is being copied
            torch.cuda.synchronize()
        assert e.stats()["precleaned_bytes_total"] >= 2 * size
        t.add_(1)
        torch.cuda.synchronize()
        added = int(t[0].item())
        r = e.evict(0)
        assert r["clean_bytes"] >= size and r["bytes"] + r["clean_bytes"] + r["elided_bytes"] == 2 * size   # `quiet` was not copied again
        assert r["bytes"] > 0                                                                            # `busy` had changed
        e.fetch_all()
        assert e.pattern_verify(quiet, size // 8, first_index=3, seed=8) == 0
        assert bool((t == torch.arange(size // 8, device="cuda", dtype=torch.int64) + added).all().item())
        del t
        e.free(quiet); e.free(busy)


@pytest.mark.parametrize("warps,stages,tile_kib", [(1, 2, 16), (1, 6, 32), (4, 3, 16), (8, 3, 8), (2, 4, 24), (1, 3, 64)])
def test_tma_ring_geometries_are_all_exact(torch_cuda, artefacts, warps, stages, tile_kib):
    """Every ring geometry the engine accepts (warps x stages x tile <= 200 KiB of shared memory) moves bytes
    identically; tiles that do not divide a slab (24 KiB) exercise the ragged last tile of each descriptor."""
    torch = torch_cuda
    from nvshare_b200 import engine as E
    size = 96 * MiB
    src = torch.empty(size, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(size, dtype=torch.uint8, device="cuda")
    with E.Engine(tma_warps=warps, tma_stages=stages, tma_tile_bytes=tile_kib << 10, prepin=0) as e:
        e.pattern_fill(src.data_ptr(), size // 8, first_index=5, seed=warps * 100 + stages)
        e.copy_slabs([(src.data_ptr() + o, dst.data_ptr() + o, SLAB) for o in range(0, size, SLAB)], variant="tma", grid=37)
        assert e.pattern_verify(dst.data_ptr(), size // 8, first_index=5, seed=warps * 100 + stages) == 0
    assert torch.equal(src, dst)


def test_torch_can_use_engine_memory(torch_cuda, engine):
    """Memory handed out by nvs_alloc behaves like cuMemAlloc memory for CUDA
    libraries: wrap it with torch via the CUDA array interface and compute."""
    torch = torch_cuda
    n = 1 << 24
    p = engine.alloc(n * 4)
    engine.fetch_all()

    class Raw:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}

    t = torch.as_tensor(Raw(p, n), device="cuda")
    t.fill_(1.0)
    torch.cuda.synchronize()
    engine.evict(0)
    engine.fetch_all()
    assert float((t + t).sum().item()) == 2.0 * n                                     # the add test's exact value
    del t
    engine.free(p)


def test_host_io_upload_and_readback_without_the_gpu(torch_cuda, engine, oracle):
    """SURVEY 8f rank 3 on the real driver: data uploaded with nvs_host_io into an
    allocation that has never been on the GPU arrives in HBM with the next fetch
    (checked by the device-side verifier), bytes nobody wrote read 0, and after
    an eviction the range can be read back from the backing copy, bit-exact."""
    torch = torch_cuda
    size = 1 * GiB + 6 * MiB
    words = size // 8
    lo_words = (300 * MiB + 8) // 8                     # upload [lo, size): slabs before it stay untouched
    host = np.empty(words, dtype=np.uint64)
    oracle.oracle_pattern_fill(host.ctypes.data, words, 11, 77)
    p = engine.alloc(size + 64 * MiB)                   # and a tail nobody writes either
    free0, _ = torch.cuda.mem_get_info()
    assert engine.host_io(p + lo_words * 8, host.ctypes.data + lo_words * 8, (words - lo_words) * 8, True) == 0
    free1, _ = torch.cuda.mem_get_info()
    assert abs(free1 - free0) < 64 * MiB                # no HBM was mapped for it
    st = engine.stats()
    assert st["resident_bytes"] == 0 and st["host_io_bytes_total"] == (words - lo_words) * 8
    rep = engine.fetch_all()
    assert rep["bytes"] <= size - 300 * MiB + 2 * MiB   # untouched slabs were not moved ...
    assert engine.pattern_verify(p + lo_words * 8, words - lo_words, first_index=11 + lo_words, seed=77) == 0

    class Raw:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}

    # chunk 0 was never touched at all and is plain fresh memory (undefined, like cuMemAlloc's);
    # the untouched slabs of chunks that DID get a backing copy must not show stale pool pages
    head = torch.as_tensor(Raw(p + 256 * MiB, 44 * MiB // 8), device="cuda")
    tail = torch.as_tensor(Raw(p + size, 64 * MiB // 8), device="cuda")
    assert int(head.abs().max().item()) == 0 and int(tail.abs().max().item()) == 0     # ... and read 0
    del head, tail
    engine.evict(0)
    back = np.full(words - lo_words, 0xEE, dtype=np.uint64)
    assert engine.host_io(p + lo_words * 8, back.ctypes.data, back.nbytes, False) == 0
    assert oracle.oracle_pattern_mismatches(back.ctypes.data, len(back), 11 + lo_words, 77) == 0
    engine.fetch_all()
    assert engine.host_io(p, back.ctypes.data, 4096, False) == -9                      # resident: device path only
    engine.free(p)
