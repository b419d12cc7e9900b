"""ctypes mirror of include/nvshare_engine.h (libnvs_engine.so).

Host-side plumbing only: every call lands in the C engine, which launches the
sm_90a slab-copy kernels.  There is no Python or CPU fallback here -- if the
shared library is missing or fails to initialise, these functions raise.

Reference interface mirrored: the engine stands where the reference has the
single call real_cuMemAllocManaged() (src/hook.c:673) plus the UVM driver; see
include/nvshare_engine.h for the per-function mapping.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_BUILD = Path(__file__).resolve().parent / "_build"
SLAB = 2 << 20
COPY_TMA, COPY_LDG, COPY_CE = 0, 1, 2
VARIANTS = {"tma": COPY_TMA, "ldg": COPY_LDG, "ce": COPY_CE}
NVS_MAX_PEERS = 7


class CopyDesc(C.Structure):
    _fields_ = [("src", C.c_uint64), ("dst", C.c_uint64), ("bytes", C.c_uint64), ("tag", C.c_uint64)]


class EngineConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("resolve", C.c_void_p),
        ("chunk_bytes", C.c_uint64), ("small_alloc_bytes", C.c_uint64), ("batch_bytes", C.c_uint64),
        ("host_arena_bytes", C.c_uint64), ("evict_variant", C.c_uint32), ("fetch_variant", C.c_uint32),
        ("copy_grid", C.c_uint32), ("tma_warps", C.c_uint32), ("tma_stages", C.c_uint32),
        ("tma_tile_bytes", C.c_uint32), ("ldg_threads", C.c_uint32), ("oom_wait_ms", C.c_uint32),
        ("prepin", C.c_uint32), ("n_peers", C.c_int32), ("peers", C.c_int32 * NVS_MAX_PEERS),
        ("peer_capacity_bytes", C.c_uint64), ("stats_path", C.c_char_p),
        ("pressure_cb", C.c_void_p), ("pressure_user", C.c_void_p),
        ("shared_pool_path", C.c_char_p), ("shared_pool_bytes", C.c_uint64), ("elide_constant", C.c_uint32),
        ("burst_bytes", C.c_uint64), ("retain", C.c_uint32), ("peer_evict_variant", C.c_uint32),
        ("peer_fetch_variant", C.c_uint32), ("preclean", C.c_uint32),
    ]


class XferReport(C.Structure):
    _fields_ = [
        ("bytes", C.c_uint64), ("slabs", C.c_uint64), ("chunks", C.c_uint64), ("launches", C.c_uint64),
        ("wall_ms", C.c_double), ("copy_ms", C.c_double), ("map_ms", C.c_double), ("wait_ms", C.c_double),
        ("host_bytes", C.c_uint64), ("peer_bytes", C.c_uint64), ("elided_bytes", C.c_uint64),
        ("clean_bytes", C.c_uint64), ("ce_calls", C.c_uint64), ("scanned_bytes", C.c_uint64), ("scan_ms", C.c_double),
        ("scan_launches", C.c_uint64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "n_allocs", "requested_bytes", "va_bytes", "resident_bytes", "swapped_bytes", "unbacked_bytes",
        "passthrough_bytes", "host_pool_bytes", "host_pool_used", "peer_pool_bytes", "peer_pool_used",
        "n_evicts", "n_fetches", "evicted_bytes_total", "fetched_bytes_total", "kernel_launches_total",
        "host_io_bytes_total", "retained_bytes", "clean_skipped_bytes_total", "stolen_slabs_total", "ce_calls_total", "precleaned_bytes_total")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class GpuAccount(C.Structure):
    """nvs_gpu_account (include/nvshare_engine.h): one GPU's row of the cross-process ledger."""
    _fields_ = [("tracked", C.c_int32), ("device", C.c_int32)] + [(n, C.c_uint64) for n in (
        "total_bytes", "reserve_bytes", "lent_bytes", "max_own_bytes", "my_lent_bytes", "my_own_bytes", "refusals")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ScanOut(C.Structure):
    _fields_ = [("value", C.c_uint64), ("is_const", C.c_uint64), ("h0", C.c_uint64), ("h1", C.c_uint64)]


class EngineError(RuntimeError):
    def __init__(self, rc, what, text):
        super().__init__(f"{what} failed: {text} (rc={rc})")
        self.rc = rc


def lib_path() -> Path:
    return Path(os.environ.get("NVS_ENGINE_LIB", _BUILD / "libnvs_engine.so"))


_lib = None


def load():
    """dlopen libnvs_engine.so (fails loudly if it was not built)."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not p.exists():
        raise FileNotFoundError(f"{p} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(str(p), mode=C.RTLD_GLOBAL)
    P = C.POINTER
    lib.nvs_engine_default_config.argtypes = [P(EngineConfig)]
    lib.nvs_engine_create.argtypes = [P(EngineConfig), P(C.c_void_p)]
    lib.nvs_engine_destroy.argtypes = [C.c_void_p]
    lib.nvs_engine_destroy.restype = None
    lib.nvs_alloc.argtypes = [C.c_void_p, P(C.c_uint64), C.c_uint64]
    lib.nvs_free.argtypes = [C.c_void_p, C.c_uint64]
    lib.nvs_set_resident_mode.argtypes = [C.c_void_p, C.c_int]
    lib.nvs_set_resident_mode.restype = None
    lib.nvs_fetch_all.argtypes = [C.c_void_p, P(XferReport)]
    lib.nvs_evict.argtypes = [C.c_void_p, C.c_uint64, P(XferReport)]
    lib.nvs_evict_best_effort.argtypes = [C.c_void_p, C.c_uint64, P(XferReport)]
    lib.nvs_get_stats.argtypes = [C.c_void_p, P(Stats)]
    lib.nvs_gpu_account_query.argtypes = [C.c_void_p, C.c_int, P(GpuAccount)]
    lib.nvs_gpu_lent_bytes.argtypes = [C.c_void_p]
    lib.nvs_gpu_lent_bytes.restype = C.c_uint64
    lib.nvs_host_io.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int]
    lib.nvs_touch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    lib.nvs_copy_slabs.argtypes = [C.c_void_p, P(CopyDesc), C.c_uint32, C.c_uint32, C.c_uint32, P(C.c_float)]
    lib.nvs_scan_slabs.argtypes = [C.c_void_p, P(CopyDesc), C.c_uint32, C.c_int, P(ScanOut), P(C.c_float)]
    lib.nvs_pattern_fill.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64]
    lib.nvs_pattern_verify.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, P(C.c_uint64)]
    lib.nvs_strerror.argtypes = [C.c_int]
    lib.nvs_strerror.restype = C.c_char_p
    lib.nvs_engine_version.restype = C.c_char_p
    _lib = lib
    return lib


def _check(rc, what):
    if rc != 0:
        raise EngineError(rc, what, load().nvs_strerror(rc).decode())


def default_config() -> EngineConfig:
    cfg = EngineConfig()
    _check(load().nvs_engine_default_config(C.byref(cfg)), "nvs_engine_default_config")
    return cfg


class Engine:
    """One swap engine bound to the CUDA context current on the creating thread."""

    def __init__(self, cfg: EngineConfig | None = None, **overrides):
        lib = load()
        cfg = cfg or default_config()
        for k, v in overrides.items():
            if k in ("evict_variant", "fetch_variant", "peer_evict_variant", "peer_fetch_variant") and isinstance(v, str):
                v = VARIANTS[v]
            if k == "peers" and v == "auto":          # NVS_PEERS_AUTO: every other visible GPU this one can reach
                cfg.n_peers = -1
                continue
            if k == "peers":
                cfg.n_peers = len(v)
                for i, d in enumerate(v):
                    cfg.peers[i] = d
                continue
            if k in ("stats_path", "shared_pool_path") and isinstance(v, str):
                v = v.encode()
            setattr(cfg, k, v)
        self.cfg = cfg
        self._h = C.c_void_p()
        _check(lib.nvs_engine_create(C.byref(cfg), C.byref(self._h)), "nvs_engine_create")

    def close(self):
        if self._h:
            load().nvs_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def alloc(self, nbytes: int) -> int:
        out = C.c_uint64()
        _check(load().nvs_alloc(self._h, C.byref(out), nbytes), "nvs_alloc")
        return out.value

    def free(self, dptr: int):
        _check(load().nvs_free(self._h, dptr), "nvs_free")

    def set_resident_mode(self, holds_lock: bool):
        load().nvs_set_resident_mode(self._h, int(holds_lock))

    def fetch_all(self) -> dict:
        rep = XferReport()
        _check(load().nvs_fetch_all(self._h, C.byref(rep)), "nvs_fetch_all")
        return rep.as_dict()

    def evict(self, min_bytes: int = 0) -> dict:
        rep = XferReport()
        _check(load().nvs_evict(self._h, min_bytes, C.byref(rep)), "nvs_evict")
        return rep.as_dict()

    def evict_best_effort(self, min_bytes: int = 0) -> dict:
        rep = XferReport()
        _check(load().nvs_evict_best_effort(self._h, min_bytes, C.byref(rep)), "nvs_evict_best_effort")
        return rep.as_dict()

    def stats(self) -> dict:
        st = Stats()
        _check(load().nvs_get_stats(self._h, C.byref(st)), "nvs_get_stats")
        return st.as_dict()

    def gpu_account(self, which: int = -1) -> dict:
        """which = -1: the GPU this engine computes on; i >= 0: peer i of the configuration."""
        acc = GpuAccount()
        _check(load().nvs_gpu_account_query(self._h, which, C.byref(acc)), "nvs_gpu_account_query")
        return acc.as_dict()

    def gpu_lent_bytes(self) -> int:
        return load().nvs_gpu_lent_bytes(self._h)

    def touch(self, dptr: int, nbytes: int):
        _check(load().nvs_touch(self._h, dptr, nbytes), "nvs_touch")

    def host_io(self, dptr: int, host_ptr: int, nbytes: int, to_device: bool) -> int:
        """nvs_host_io: 0 = served from / into the backing copy, NVS_E_NOT_OURS / NVS_E_NOT_SWAPPED =
        the caller must use the device path; anything else raises."""
        rc = load().nvs_host_io(self._h, dptr, host_ptr, nbytes, 1 if to_device else 0)
        if rc not in (0, -2, -9):
            _check(rc, "nvs_host_io")
        return rc

    def copy_slabs(self, descs, variant="tma", grid=0) -> float:
        """descs: iterable of (src, dst, nbytes). Returns CUDA-event milliseconds."""
        descs = list(descs)
        arr = (CopyDesc * max(len(descs), 1))()
        for i, (s, d, b) in enumerate(descs):
            arr[i].src, arr[i].dst, arr[i].bytes, arr[i].tag = s, d, b, i
        ms = C.c_float()
        v = VARIANTS[variant] if isinstance(variant, str) else variant
        _check(load().nvs_copy_slabs(self._h, arr, len(descs), v, grid, C.byref(ms)), "nvs_copy_slabs")
        return ms.value

    def pattern_fill(self, addr: int, n_words: int, first_index: int = 0, seed: int = 1):
        _check(load().nvs_pattern_fill(self._h, addr, n_words, first_index, seed), "nvs_pattern_fill")

    def pattern_verify(self, addr: int, n_words: int, first_index: int = 0, seed: int = 1) -> int:
        bad = C.c_uint64()
        _check(load().nvs_pattern_verify(self._h, addr, n_words, first_index, seed, C.byref(bad)),
               "nvs_pattern_verify")
        return bad.value


def scan_slabs(engine: Engine, descs, want_hash=True, with_ms=False):
    """nvs_scan_slabs: run the sm_90a scan/hash kernel over (src, _, nbytes) ranges."""
    descs = list(descs)
    arr = (CopyDesc * max(len(descs), 1))()
    for i, (s, _d, b) in enumerate(descs):
        arr[i].src, arr[i].dst, arr[i].bytes, arr[i].tag = s, 0, b, i
    out = (ScanOut * max(len(descs), 1))()
    ms = C.c_float()
    _check(load().nvs_scan_slabs(engine._h, arr, len(descs), 1 if want_hash else 0, out, C.byref(ms)), "nvs_scan_slabs")
    res = [{"value": o.value, "is_const": o.is_const, "h0": o.h0, "h1": o.h1} for o in out[:len(descs)]]
    return (res, ms.value) if with_ms else res
