"""The kernels that decide which bytes are NOT copied (nvs_slab_scan: same-filled test, content hash, fused
copy + hash; nvs_slab_splat: re-creation of an elided slab) and the copy kernels, at the inputs where a subtly
wrong kernel loses data without crashing: 64-bit values whose 32-bit halves differ, slabs that differ only in
their last 32 KiB tile, descriptors one vector either side of a tile, many descriptors per CTA, destinations
scattered between guard bands.

Every case runs twice: against oracle/fake_cuda.c on the CPU (unmarked) and against the sm_90a kernels on an
H100 (marked gpu; torch only provides the context and the buffers).  Expected values always come from the
oracle (oracle/nvshare_oracle.c: oracle_slab_is_const, oracle_slab_hash, oracle_slab_move) applied to host
copies of the bytes, never from the kernel under test."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from nvs_testlib import FAKE_DIR, ORACLE

MiB = 1 << 20
SLAB = 2 * MiB
TILE = 32 << 10                  # the scan's early-exit granularity: 256 threads x 8 vectors x 16 bytes
WORDS = SLAB // 8
SENTINEL = 0xA5
V = 0x0123456789ABCDEF
M64 = (1 << 64) - 1
NVS_E_BAD_ARG = -3


def swap_halves(x):
    return ((x << 32) | (x >> 32)) & M64


CONST_VALUES = [0, M64, 1 << 63, 0x00000001_00000002, 0x00000002_00000001, 0x3F800000_3F800000]


def _libcuda_is_fake():
    """Which libcuda.so.1 this process resolves (the engine dlopens it by that name)."""
    return hasattr(C.CDLL("libcuda.so.1"), "fake_cuda_launch_count")


class Buf:
    """A buffer the kernels can address: host memory on the fake driver, HBM or pinned host on the GPU."""

    def __init__(self, be, nbytes, where="device", fill=None):
        self.nbytes = nbytes
        self.t = None
        if be.torch is None:
            self.raw = np.empty(nbytes + 256, dtype=np.uint8)
            lead = (-self.raw.ctypes.data) % 256
            self.np = self.raw[lead:lead + nbytes]
        elif where == "device":
            self.t = be.torch.empty(nbytes, dtype=be.torch.uint8, device="cuda")
            self.np = None
        else:
            self.t = be.torch.empty(nbytes, dtype=be.torch.uint8).pin_memory()
            self.np = self.t.numpy()
        self.ptr = self.np.ctypes.data if self.np is not None else self.t.data_ptr()
        assert self.ptr % 256 == 0
        self.be = be
        if fill is not None:
            self.write(0, np.full(nbytes, fill, dtype=np.uint8))

    def write(self, off, data):
        data = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
        if self.np is not None:
            self.np[off:off + data.size] = data
        else:
            self.t[off:off + data.size].copy_(self.be.torch.from_numpy(data))
            self.be.torch.cuda.synchronize()

    def read(self):
        if self.np is not None:
            return self.np.copy()
        return self.t.cpu().numpy()


class Backend:
    def __init__(self, kind, torch=None):
        self.kind, self.torch = kind, torch

    def engine(self, **kw):
        from nvshare_b200 import engine as E
        # small chunks so that a few MiB span several; no background pre-cleaning: it would write chunks back while
        # a test fills them.  The same configuration on both drivers.
        args = dict(chunk_bytes=8 * MiB, host_arena_bytes=64 * MiB, batch_bytes=24 * MiB, oom_wait_ms=300, prepin=0,
                    preclean=0)
        args.update(kw)
        return E.Engine(**args)

    def write_alloc(self, ptr, data):
        """Write host bytes into engine-allocated (resident) memory."""
        data = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
        if self.torch is None:
            C.memmove(ptr, data.ctypes.data, data.size)
            return
        self.torch.as_tensor(_Raw(ptr, data.size), device="cuda").copy_(self.torch.from_numpy(data))
        self.torch.cuda.synchronize()

    def read_alloc(self, ptr, nbytes):
        if self.torch is None:
            return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr)).copy()
        return self.torch.as_tensor(_Raw(ptr, nbytes), device="cuda").cpu().numpy()


class _Raw:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}


@pytest.fixture(scope="module", params=["fake", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request, artefacts):
    if request.param == "fake":
        lib = C.CDLL(str(FAKE_DIR / "libcuda.so.1"), mode=C.RTLD_GLOBAL)
        if not _libcuda_is_fake():
            pytest.skip("this process already uses the real CUDA driver")
        assert lib.cuInit(0) == 0
        ctx = C.c_void_p()
        assert lib.cuDevicePrimaryCtxRetain(C.byref(ctx), 0) == 0
        assert lib.cuCtxSetCurrent(ctx) == 0
        b = Backend("fake")
        b.fake = lib
        return b
    import torch
    if _libcuda_is_fake():
        pytest.skip("this process has loaded the fake CUDA driver")
    if not torch.cuda.is_available():
        pytest.skip("these tests need a GPU")
    torch.cuda.init()
    torch.zeros(1, device="cuda")          # makes the primary context current on this thread
    return Backend("gpu", torch)


@pytest.fixture(scope="module")
def oracle(artefacts):
    lib = C.CDLL(str(ORACLE / "liboracle.so"))
    lib.oracle_slab_is_const.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.oracle_slab_hash.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64 * 2)]
    lib.oracle_slab_move.argtypes = [C.c_void_p, C.c_uint32]
    return lib


@pytest.fixture(scope="module")
def eng(be):
    e = be.engine()
    yield e
    e.close()


def o_const(oracle, host, off, nbytes):
    """(is_const, value) of host[off:off+nbytes] by the oracle; value = the first word when not const."""
    v = C.c_uint64()
    k = oracle.oracle_slab_is_const(host.ctypes.data + off, nbytes, C.byref(v))
    return k, (v.value if k else int(host[off:off + 8].view(np.uint64)[0]))


def o_hash(oracle, host, off, nbytes):
    h = (C.c_uint64 * 2)()
    oracle.oracle_slab_hash(host.ctypes.data + off, nbytes, C.byref(h))
    return h[0], h[1]


def o_move(oracle, pieces, src_host, dst_host):
    """oracle_slab_move of (src_off, dst_off, nbytes) pieces on host copies; returns the expected dst."""
    from nvshare_b200.engine import CopyDesc
    want = dst_host.copy()
    arr = (CopyDesc * len(pieces))()
    for i, (s, d, n) in enumerate(pieces):
        arr[i].src, arr[i].dst, arr[i].bytes = src_host.ctypes.data + s, want.ctypes.data + d, n
    oracle.oracle_slab_move(arr, len(pieces))
    return want


def scatter(rng, sizes, guard=4096):
    """Destination offsets for pieces of the given sizes, in a random order, each with a guard band of at least
    `guard` bytes (and a random multiple of 16 more) before it, and one after the last.  Returns (offsets, total)."""
    offs = [0] * len(sizes)
    at = guard
    for i in rng.permutation(len(sizes)):
        offs[i] = at
        at += (sizes[i] + 15) & ~15
        at += guard + 16 * int(rng.integers(0, 64))
    return offs, at


# ------------------------------------------------------------------ 1. same-filled detection --


def near_constant_slabs():
    """(name, 2 MiB slab as uint64 words) pairs: constant ones, and ones that are constant but for one place."""
    out = [(f"const {v:#018x}", np.full(WORDS, v, dtype=np.uint64)) for v in CONST_VALUES + [V]]
    tile_words = TILE // 8
    changes = {"word 1 (same vector as word 0)": 1, "last word": WORDS - 1, "first word of tile 1": tile_words,
               "first word of tile 31": 31 * tile_words, "first word of tile 63": 63 * tile_words}
    for name, i in changes.items():
        w = np.full(WORDS, V, dtype=np.uint64)
        w[i] = V ^ 0x10
        out.append((name, w))
    w = np.full(WORDS, V, dtype=np.uint64)
    w[17 * tile_words + 2 * 777 + 1] = V ^ (1 << 63)        # an odd word's high half: the `w` lane of its vector
    out.append(("odd word, top bit", w))
    w = np.full(WORDS, V, dtype=np.uint64)
    w[1::2] = swap_halves(V)                                 # 32-bit periodic, not constant in 64 bits
    out.append(("halves alternate", w))
    return out


def test_same_filled_detection_matches_the_oracle(be, eng, oracle):
    from nvshare_b200 import engine as E
    slabs = near_constant_slabs()
    host = np.concatenate([w for _, w in slabs]).view(np.uint8)
    src = Buf(be, host.size)
    src.write(0, host)
    descs = [(src.ptr + i * SLAB, 0, SLAB) for i in range(len(slabs))]
    full = E.scan_slabs(eng, descs, want_hash=True)
    quick = E.scan_slabs(eng, descs, want_hash=False)
    n_const = 0
    for i, (name, _) in enumerate(slabs):
        k, v = o_const(oracle, host, i * SLAB, SLAB)
        n_const += k
        for how, o in (("full scan", full[i]), ("early-exit scan", quick[i])):
            assert (o["is_const"], o["value"]) == (k, v), f"{name}: {how}"
        assert (full[i]["h0"], full[i]["h1"]) == o_hash(oracle, host, i * SLAB, SLAB), name
        assert quick[i]["h0"] == 0 and quick[i]["h1"] == 0, name
    assert n_const == len(CONST_VALUES) + 1                  # the oracle agrees with how the slabs were built


# --------------------------------------------------------------------- 2. hash, bit for bit --


HASH_SIZES = [16, 32, 4080, 4096, 4112, 32752, 32768, 32784, SLAB - 16, SLAB]


def test_hash_matches_the_oracle_at_every_size_and_misaligned_sources(be, eng, oracle):
    """Sources 16-byte aligned but never 256-byte aligned; sizes one vector either side of a 4 KiB page and of a
    32 KiB tile, and of a slab."""
    from nvshare_b200 import engine as E
    rng = np.random.default_rng(21)
    offs, at = [], 256
    for n in HASH_SIZES:
        offs.append(at + 16 * int(rng.integers(1, 16)))     # == 16..240 mod 256
        at = (offs[-1] + n + 255) & ~255
    host = rng.integers(0, 256, at, dtype=np.uint8)
    src = Buf(be, at)
    src.write(0, host)
    descs = [(src.ptr + o, 0, n) for o, n in zip(offs, HASH_SIZES)]
    assert all((s % 256) != 0 for s, _, _ in descs)
    out = E.scan_slabs(eng, descs, want_hash=True)
    for o, n, r in zip(offs, HASH_SIZES, out):
        assert (r["h0"], r["h1"]) == o_hash(oracle, host, o, n), f"{n} bytes at +{o}"
        assert (r["is_const"], r["value"]) == o_const(oracle, host, o, n), f"{n} bytes at +{o}"


def test_hash_with_many_descriptors_per_cta(be, eng, oracle):
    """1536 descriptors of mixed sizes: the scan grid is at most 4 CTAs per SM (528 on an H100), so every CTA takes
    several and carries its shared state from one descriptor to the next.  Same-filled ones are mixed in."""
    from nvshare_b200 import engine as E
    rng = np.random.default_rng(22)
    n = 1536
    size = 8 * MiB
    host = rng.integers(0, 256, size, dtype=np.uint8)
    host[3 * MiB:4 * MiB] = 0x3C                             # a same-filled region some descriptors fall into
    host[5 * MiB:6 * MiB].view(np.uint64)[:] = 0x00000001_00000002
    menu = [16, 32, 4080, 4096, 4112, 32752, 32768, 32784, 65536]
    sizes = [int(rng.choice(menu)) if rng.random() < 0.7 else 16 * int(rng.integers(1, 8192)) for _ in range(n)]
    offs = [16 * int(rng.integers(0, (size - s) // 16)) for s in sizes]
    offs[:16] = [3 * MiB + 4096 * k for k in range(8)] + [5 * MiB + 16 * 1024 * k for k in range(8)]
    sizes[:16] = [4096] * 16
    src = Buf(be, size)
    src.write(0, host)
    descs = [(src.ptr + o, 0, s) for o, s in zip(offs, sizes)]
    out = E.scan_slabs(eng, descs, want_hash=True)
    for i, (o, s, r) in enumerate(zip(offs, sizes, out)):
        assert (r["h0"], r["h1"]) == o_hash(oracle, host, o, s), f"descriptor {i}: {s} bytes at +{o}"
        assert (r["is_const"], r["value"]) == o_const(oracle, host, o, s), f"descriptor {i}: {s} bytes at +{o}"
    assert sum(r["is_const"] for r in out) >= 16


# ------------------------------------------------------------------- 3. fused copy + hash --


@pytest.mark.parametrize("want_hash", [0, 1])
@pytest.mark.parametrize("where", ["device", "pinned"])
def test_fused_copy_and_hash(be, eng, oracle, where, want_hash):
    """nvs_scan_slabs with a destination, as the pre-cleaner runs it (its destination is pinned host memory): every
    range lands in full at its permuted destination and nothing else is written; the hash, reported whatever
    want_hash says, is the oracle's hash of the bytes in dst; a slab that differs only in its last tile is copied
    in full even without a hash."""
    from nvshare_b200 import engine as E
    rng = np.random.default_rng(30 + want_hash)
    sizes = [SLAB, SLAB - 16, SLAB, SLAB, 32784, 32768, 4112, 16, SLAB]
    src_offs = [16 + sum(sizes[:i]) for i in range(len(sizes))]
    host = rng.integers(0, 256, 16 + sum(sizes), dtype=np.uint8)
    const_at = src_offs[2]
    host[const_at:const_at + SLAB].view(np.uint64)[:] = 0x00000002_00000001          # same-filled
    late_at = src_offs[3]
    late = host[late_at:late_at + SLAB].view(np.uint64)
    late[:] = V
    late[WORDS - 1] = swap_halves(V)                                                  # differs in its last tile only
    src = Buf(be, host.size)
    src.write(0, host)
    dst_offs, total = scatter(rng, sizes)
    dst = Buf(be, total, where=where, fill=SENTINEL)
    pieces = list(zip(src_offs, dst_offs, sizes))
    out = E.scan_slabs(eng, [(src.ptr + s, dst.ptr + d, n) for s, d, n in pieces], want_hash=bool(want_hash), copy=True)
    got = dst.read()
    want = o_move(oracle, pieces, host, np.full(total, SENTINEL, dtype=np.uint8))
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} bytes differ, first at dst+{bad[0]}"
    for (s, d, n), r in zip(pieces, out):
        assert (r["h0"], r["h1"]) == o_hash(oracle, got, d, n), f"{n} bytes at dst+{d}"
        assert (r["is_const"], r["value"]) == o_const(oracle, got, d, n), f"{n} bytes at dst+{d}"
    assert [r["is_const"] for r in out] == [0, 0, 1, 0, 0, 0, 0, 0, 0]


def test_misaligned_scan_destination_is_refused(eng, be, oracle):
    """A dst that is not 16-byte aligned is refused before anything is launched (the kernel stores 16-byte
    vectors).  Fake driver only: nothing misaligned is ever handed to a real GPU."""
    from nvshare_b200 import engine as E
    if be.kind != "fake":
        pytest.skip("checked on the fake driver only")
    src = Buf(be, 4096)
    src.write(0, np.arange(4096, dtype=np.uint32).view(np.uint8)[:4096])
    dst = Buf(be, 8192, fill=SENTINEL)
    launches = be.fake.fake_cuda_launch_count()
    for off in (1, 8, 4095):
        with pytest.raises(E.EngineError) as ex:
            E.scan_slabs(eng, [(src.ptr, 0, 4096), (src.ptr, dst.ptr + off, 4096)], want_hash=True, copy=True)
        assert ex.value.rc == NVS_E_BAD_ARG
    assert be.fake.fake_cuda_launch_count() == launches
    assert (dst.read() == SENTINEL).all()
    # dst = 0 is a scan; copy=False leaves any dst out
    assert E.scan_slabs(eng, [(src.ptr, 0, 4096)])[0]["h0"] == o_hash(oracle, src.read(), 0, 4096)[0]
    assert E.scan_slabs(eng, [(src.ptr, dst.ptr + 8, 4096)])[0]["h0"] == o_hash(oracle, src.read(), 0, 4096)[0]
    assert (dst.read() == SENTINEL).all()


# ------------------------------------------------------------------------- 4. copy kernels --


COPY_CASES = [("tma", 32 << 10), ("tma", 24 << 10), ("ldg", 32 << 10), ("ce", 32 << 10)]


@pytest.mark.parametrize("variant,tile", COPY_CASES, ids=["tma", "tma-24k", "ldg", "ce"])
def test_copy_kernels_write_exactly_their_destinations(be, oracle, variant, tile):
    """Pieces one vector either side of a tile and of a slab, scattered to permuted destinations between guard
    bands of sentinel bytes; more descriptors than grid x warps x stages.  The whole destination, guards
    included, must equal oracle_slab_move's."""
    rng = np.random.default_rng(40 + tile // 1024)
    grid = 4
    menu = [16, tile - 16, tile, tile + 16, SLAB - 16, SLAB]
    sizes = menu * 8
    if variant == "ldg":
        sizes += [16 * int(rng.integers(0, 4)) + r for r in range(1, 16)] + [tile + r for r in (1, 7, 15)]
    sizes = [int(s) for s in rng.permutation(sizes)]
    src_offs, at = [], 0
    for s in sizes:
        src_offs.append(at)
        at += (s + 15) & ~15
    host = rng.integers(0, 256, at, dtype=np.uint8)
    dst_offs, total = scatter(rng, sizes)
    pieces = list(zip(src_offs, dst_offs, sizes))
    want = o_move(oracle, pieces, host, np.full(total, SENTINEL, dtype=np.uint8))
    e = be.engine(tma_tile_bytes=tile)
    try:
        assert len(pieces) > grid * e.cfg.tma_warps * e.cfg.tma_stages
        src = Buf(be, at)
        src.write(0, host)
        dst = Buf(be, total, fill=SENTINEL)
        e.copy_slabs([(src.ptr + s, dst.ptr + d, n) for s, d, n in pieces], variant=variant, grid=grid)
        got = dst.read()
    finally:
        e.close()
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} bytes differ, first at dst+{bad[0]}"


# ---------------------------------------------------------------- 5. splat, through the engine --


def splat_slabs():
    """The slabs of one allocation: every constant value of case 1 in a slab of its own, interleaved with
    position-dependent ones, plus slabs that are constant except in their last tile."""
    rng = np.random.default_rng(50)
    slabs = []
    for v in CONST_VALUES + [V]:
        slabs.append(np.full(WORDS, v, dtype=np.uint64))
        slabs.append(rng.integers(0, 1 << 63, WORDS, dtype=np.uint64))
    for v in (0, swap_halves(V)):
        w = np.full(WORDS, v, dtype=np.uint64)
        w[WORDS - 1 - 3 * 64] ^= 1 << 40                     # in the last 32 KiB tile only
        slabs.append(w)
    return np.concatenate(slabs).view(np.uint8)


@pytest.mark.parametrize("retain", [1, 0])
def test_same_filled_slabs_survive_eviction_and_fetch(be, oracle, retain):
    """Evict and fetch an allocation of several chunks (the last one partial): same-filled slabs are elided and
    re-created by the splat, everything else is copied, and the allocation comes back bit for bit.  retain=0
    evicts with the early-exit scan (no hashes), retain=1 with the full one."""
    host = splat_slabs()
    n_slabs = host.size // SLAB
    want_const = sum(o_const(oracle, host, i * SLAB, SLAB)[0] for i in range(n_slabs))
    assert want_const == len(CONST_VALUES) + 1
    e = be.engine(retain=retain)
    try:
        p = e.alloc(host.size)
        e.fetch_all()
        be.write_alloc(p, host)
        r = e.evict(0)
        assert e.stats()["resident_bytes"] == 0
        assert r["elided_bytes"] == want_const * SLAB and r["bytes"] == (n_slabs - want_const) * SLAB
        r = e.fetch_all()
        assert r["elided_bytes"] == want_const * SLAB and r["bytes"] == (n_slabs - want_const) * SLAB
        got = be.read_alloc(p, host.size)
        bad = np.flatnonzero(got != host)
        assert bad.size == 0, f"{bad.size} bytes differ, first in slab {bad[0] // SLAB} at +{bad[0] % SLAB}"
        e.free(p)
    finally:
        e.close()
