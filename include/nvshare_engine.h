/*
 * nvshare_engine.h -- C-ABI of the H100 swap engine: the explicit
 * prefetch/evict data path that replaces the reference's one-line data path
 *
 *     real_cuMemAllocManaged(dptr, bytesize, CU_MEM_ATTACH_GLOBAL)
 *                                              (reference src/hook.c:673)
 *
 * and everything NVIDIA's UVM driver does behind it (GPU page fault ->
 * migrate 4 KiB..2 MiB -> LRU-evict some context's pages).  Exported by
 * libnvshare.so (where the LD_PRELOAD hook and the client runtime are its only
 * callers) and by libnvs_engine.so (the same object without the interposer,
 * for ctypes-driven parity tests and bench.py).  Plain C: pointers and sizes
 * only, no CUDA SDK types, no torch types.
 *
 * Reference interface each entry point replaces (file:line in /root/reference):
 *   nvs_alloc        src/hook.c:646-682  cuMemAlloc hook body (after the cap
 *                    check, which stays in the hook): cuMemAllocManaged +
 *                    insert_cuda_allocation (src/hook.c:273-288)
 *   nvs_free         src/hook.c:685-695  real_cuMemFree + remove_cuda_allocation
 *                    (src/hook.c:291-305)
 *   nvs_fetch_all    what UVM does implicitly after LOCK_OK opens the gate
 *                    (src/client.c:298-307 -> first touch faults); here it runs
 *                    BEFORE own_lock is set
 *   nvs_evict        what UVM does implicitly while another context faults its
 *                    pages in; here it runs after cuda_sync_context() on
 *                    DROP_LOCK (src/client.c:308-317) and on early release
 *                    (src/client.c:472-476)
 *   nvs_evict_announce
 *                    no counterpart: tells the next holder's fetch (through the shared pool
 *                    header) that HBM is about to be released for it
 *   nvs_evict_best_effort
 *                    no counterpart: eviction as a favour to the client that is
 *                    mapping (memory-pressure hint on the wire); never waits for
 *                    backing space
 *   nvs_host_io      src/hook.c:878-938 cuMemcpyDtoH/HtoD{,Async} hook bodies, for the
 *                    case the reference cannot have: the device range is not on
 *                    the GPU at all (swapped out / never materialised), so the
 *                    copy is host memory -> pinned host backing and needs
 *                    neither the GPU nor its lock (SURVEY 8f rank 3)
 *   nvs_get_stats    no counterpart (the reference has no counters, SURVEY 5)
 *   nvs_gpu_account_query / nvs_gpu_lent_bytes
 *                    src/hook.c:77-78, 662 (sum_allocated and the cap check), extended from
 *                    "this process, device 0" to "every process, per GPU" (SURVEY 8e)
 *   nvs_touch        no counterpart (recency hint from the hooked cuMemcpy / cuMemset calls)
 *   nvs_copy_slabs / nvs_scan_slabs / nvs_pattern_fill / nvs_pattern_verify
 *                    no counterpart: raw access to the sm_90a kernels for the
 *                    parity tests and the roofline measurement
 *
 * Return values: 0 on success, otherwise a CUresult value from the driver
 * (2 = CUDA_ERROR_OUT_OF_MEMORY, 3 = CUDA_ERROR_NOT_INITIALIZED, ...) or one
 * of the negative NVS_E_* codes below.  No device copy ever falls back to the
 * CPU: if the driver or the kernel image cannot be loaded, creation fails, and
 * bytes that are in HBM only move by the sm_90a kernels / copy engines.
 * (nvs_host_io is not such a fallback: both ends of its copies are host RAM.)
 */
#ifndef NVSHARE_ENGINE_H
#define NVSHARE_ENGINE_H

#include <stdint.h>
#include "nvs_copy_desc.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NVS_E_NOT_OURS   (-2) /* pointer was not allocated by this engine          */
#define NVS_E_BAD_ARG    (-3)
#define NVS_E_NO_DRIVER  (-4) /* libcuda.so.1 or a required entry point is missing */
#define NVS_E_NO_KERNEL  (-5) /* embedded sm_90a image failed to load             */
#define NVS_E_TIMEOUT    (-6) /* HBM did not become available in time              */
#define NVS_E_HOST_OOM   (-7) /* backing tier exhausted                            */
#define NVS_E_SHUTDOWN   (-8) /* the CUDA context is being destroyed (process exit) */
#define NVS_E_NOT_SWAPPED (-9) /* nvs_host_io: the range is not (entirely) off the GPU */

#define NVS_MAX_PEERS 7
#define NVS_PEERS_AUTO (-1)

typedef struct nvs_engine nvs_engine;

/* Resolves a driver entry point by its exported ELF name (e.g. "cuMemCreate",
 * "cuMemAlloc_v2").  libnvshare.so passes a resolver built on the REAL dlsym
 * so the engine never sees the interposed symbols. */
typedef void *(*nvs_resolve_fn)(const char *symbol);

typedef struct nvs_engine_config {
	uint32_t struct_size;        /* sizeof(nvs_engine_config), for ABI growth          */
	int32_t  device;             /* CUDA ordinal; -1 = device of the current context   */
	nvs_resolve_fn resolve;      /* NULL = dlopen("libcuda.so.1") + dlsym              */
	uint64_t chunk_bytes;        /* physical mapping unit, multiple of 2 MiB (256 MiB) */
	uint64_t small_alloc_bytes;  /* smaller requests stay plain cuMemAlloc (1 MiB)     */
	uint64_t batch_bytes;        /* pipeline batch: copy(b+1) overlaps (un)map(b)      */
	uint64_t host_arena_bytes;   /* pinned-host growth unit (1 GiB)                    */
	uint32_t evict_variant;      /* enum nvs_copy_variant                              */
	uint32_t fetch_variant;      /* enum nvs_copy_variant                              */
	uint32_t copy_grid;          /* CTAs per copy launch                               */
	uint32_t tma_warps;          /* warps per CTA (TMA variant)                        */
	uint32_t tma_stages;         /* ring depth per warp                                */
	uint32_t tma_tile_bytes;     /* bytes per stage                                    */
	uint32_t ldg_threads;        /* threads per CTA (LDG variant)                      */
	uint32_t oom_wait_ms;        /* how long fetch/alloc wait for HBM to be released   */
	uint32_t prepin;             /* 1 = grow the pinned pool in the background on alloc */
	int32_t  n_peers;            /* peer-HBM backing tier: devices, in striping order;
	                              * NVS_PEERS_AUTO = every other visible GPU this one can
	                              * reach over NVLink/PCIe P2P (NVSHARE_PEERS=auto)      */
	int32_t  peers[NVS_MAX_PEERS];
	uint64_t peer_capacity_bytes; /* per peer; 0 = none                                */
	const char *stats_path;      /* JSON lines, one per evict/fetch; NULL = off        */
	/* called (rate-limited) while a fetch/alloc waits for HBM other processes hold:
	 * `bytes` = what is still missing.  libnvshare.so turns it into a REQ_LOCK "p<MiB>". */
	void (*pressure_cb)(void *user, uint64_t bytes);
	void *pressure_user;
	/* Host backing shared by all clients of one scheduler (a file, normally in
	 * /dev/shm): host RAM then follows what is actually swapped out instead of
	 * the sum of per-process pools.  NULL = private cuMemHostAlloc arenas. */
	const char *shared_pool_path;
	uint64_t shared_pool_bytes;  /* capacity when this client creates it; 0 = one HBM */
	/* 1 = scan slabs before eviction and do not move same-filled ones (all 64-bit
	 * words equal): they are re-created on the device at fetch (nvs_slab_splat) */
	uint32_t elide_constant;
	/* a fetch that needs HBM somebody else is still releasing waits while the free HBM keeps
	 * growing and starts mapping when it has stood still for a few ms, or when this many bytes
	 * (64 GiB) are free: release and create calls of two processes must not interleave */
	uint64_t burst_bytes;
	/* 1 = keep the backing copy of a chunk after it has been fetched (as long as the pool has
	 * room: retained units are the first to be reclaimed), record a 128-bit hash per slab when a
	 * copy is written, and at the next eviction do not copy slabs whose hash is unchanged */
	uint32_t retain;
	/* copy variants for the peer-HBM tier (NVLink); evict_variant / fetch_variant above apply to
	 * the pinned-host tier (PCIe), where the copy engines beat any SM kernel by the TLP size */
	uint32_t peer_evict_variant;
	uint32_t peer_fetch_variant;
	/* 1 = while the owner holds the GPU lock, write resident chunks that have no backing copy back
	 * in the background (fused copy + hash kernel, lowest-priority stream): the link is idle then,
	 * and whatever has not changed again by the hand-off does not have to be copied on it */
	uint32_t preclean;
} nvs_engine_config;

typedef struct nvs_xfer_report {
	uint64_t bytes;        /* payload bytes moved (algorithmic: 2 MiB per slab, once) */
	uint64_t slabs;
	uint64_t chunks;       /* physical chunks (un)mapped                              */
	uint64_t launches;     /* copy kernel launches (or CE calls)                      */
	double   wall_ms;      /* whole call                                              */
	double   copy_ms;      /* CUDA-event time, first launch start -> last launch end  */
	double   map_ms;       /* host time in cuMemCreate/Map/SetAccess or Unmap/Release */
	double   wait_ms;      /* host time spent waiting for HBM (OOM retries)           */
	uint64_t host_bytes;   /* of `bytes`, how much went to / came from the host tier  */
	uint64_t peer_bytes;   /* ... the peer-HBM tier                                   */
	uint64_t elided_bytes; /* same-filled slabs: swapped without crossing the link    */
	uint64_t clean_bytes;  /* evict: slabs whose retained backing copy was still valid
	                          (hash unchanged): swapped out without being copied      */
	uint64_t ce_calls;     /* cuMemcpyAsync calls (copy engines); `launches` counts
	                          sm_90a kernel launches only                            */
	uint64_t scanned_bytes; /* bytes the scan/hash kernel read from HBM                */
	double   scan_ms;      /* CUDA-event time of the scan/hash launches               */
	uint64_t scan_launches; /* how many of `launches` were scan/hash launches          */
} nvs_xfer_report;

typedef struct nvs_stats {
	uint64_t n_allocs;
	uint64_t requested_bytes;   /* sum of sizes the application asked for            */
	uint64_t va_bytes;          /* reserved virtual range (2 MiB rounded)            */
	uint64_t resident_bytes;    /* chunks currently mapped to HBM                    */
	uint64_t swapped_bytes;     /* chunks whose only copy is in the backing tier     */
	uint64_t unbacked_bytes;    /* chunks never materialised (no copy needed)        */
	uint64_t passthrough_bytes; /* small allocations left to plain cuMemAlloc        */
	uint64_t host_pool_bytes;   /* pinned host memory owned by the pool              */
	uint64_t host_pool_used;
	uint64_t peer_pool_bytes;
	uint64_t peer_pool_used;
	uint64_t n_evicts, n_fetches;
	uint64_t evicted_bytes_total, fetched_bytes_total;
	uint64_t kernel_launches_total; /* nvs_slab_copy_* launches since creation       */
	uint64_t host_io_bytes_total;   /* nvs_host_io: bytes served from / into the backing copy */
	uint64_t retained_bytes;        /* resident chunks whose backing copy is being kept        */
	uint64_t clean_skipped_bytes_total; /* eviction bytes that did not have to be copied       */
	uint64_t stolen_slabs_total;    /* retained units this engine took over from other chunks  */
	uint64_t ce_calls_total;        /* cuMemcpyAsync calls issued by evict / fetch             */
	uint64_t precleaned_bytes_total; /* written back in the background during the owner's quantum */
} nvs_stats;

/* Fill *cfg with defaults, then apply NVSHARE_* environment overrides
 * (NVSHARE_CHUNK_MIB, NVSHARE_COPY_VARIANT, NVSHARE_COPY_GRID, NVSHARE_PEERS, ...). */
int nvs_engine_default_config(nvs_engine_config *cfg);

/* Requires a current CUDA context on the calling thread; the engine keeps using it. */
int nvs_engine_create(const nvs_engine_config *cfg, nvs_engine **out);
void nvs_engine_destroy(nvs_engine *e);

int nvs_alloc(nvs_engine *e, uint64_t *dptr, uint64_t bytes);
int nvs_free(nvs_engine *e, uint64_t dptr);
/* same, also reporting the size the application had asked for (the hook's
 * sum_allocated bookkeeping, reference src/hook.c:298) */
int nvs_free_sized(nvs_engine *e, uint64_t dptr, uint64_t *req_bytes);

/* Tell the engine whether its owner currently holds the GPU lock: new
 * allocations are materialised immediately when it does, deferred otherwise. */
void nvs_set_resident_mode(nvs_engine *e, int holds_lock);

int nvs_fetch_all(nvs_engine *e, nvs_xfer_report *rep);
/* Evict at least `min_bytes` (0 = everything) of resident chunks, least
 * recently fetched first, and release their physical HBM. */
int nvs_evict(nvs_engine *e, uint64_t min_bytes, nvs_xfer_report *rep);

/*
 * Serve a host<->device copy WITHOUT the GPU, from / into the pinned-host backing
 * copy of memory that is currently swapped out (or was never materialised).  The
 * reference has no counterpart: there every cuMemcpy* waits for the GPU lock
 * (src/hook.c:843-971) even when the data it wants is sitting in host RAM, and a
 * client that is loading its inputs keeps the GPU from the others meanwhile.
 *   to_device != 0: host -> [dptr, dptr+bytes)   (cuMemcpyHtoD*)
 *   to_device == 0: [dptr, dptr+bytes) -> host   (cuMemcpyDtoH*)
 * Returns 0 when the whole range was served.  NVS_E_NOT_OURS: the range is not
 * inside one engine allocation.  NVS_E_NOT_SWAPPED: some of it is resident in
 * HBM, backed by a peer GPU, or (reads) was never written: use the GPU path.
 * A failed call may have written part of a host->device range; the caller then
 * repeats the whole copy on the GPU path, which makes that harmless.
 */
int nvs_host_io(nvs_engine *e, uint64_t dptr, void *host, uint64_t bytes, int to_device);

/* Say that an eviction for the next holder is about to start (call it BEFORE the lock is given
 * away, nvs_evict after): the next holder's fetch then follows this engine's release progress
 * through the shared pool instead of polling the driver.  No-op without a shared pool. */
void nvs_evict_announce(nvs_engine *e);

/* Like nvs_evict, but never waits for room in the backing tier: it evicts what the
 * tier can take right now and returns 0 (possibly having moved less than asked).
 * For evictions done as a favour to another client (memory pressure) by a client
 * that may itself be about to be granted the lock: waiting there for pool units
 * that only its own next fetch would free is a deadlock. */
int nvs_evict_best_effort(nvs_engine *e, uint64_t min_bytes, nvs_xfer_report *rep);

int nvs_get_stats(nvs_engine *e, nvs_stats *out);

/*
 * Per-GPU accounting across processes and schedulers (SURVEY 8e: "peers' HBM used as backing
 * must be accounted in those GPUs' caps").  The reference counts per process and knows one GPU
 * (sum_allocated, src/hook.c:77-78, 662; device 0, src/client.c:386).  Here every engine records,
 * in one small ledger file per user and machine, the backing arenas it creates on peer GPUs
 * ("lent") and the swappable memory its owner has allocated on the GPU it computes on ("own");
 * a peer arena is only created while  lent + arena <= total - reserve - largest own  on that GPU,
 * and the hook shrinks the cuMemGetInfo / cuMemAlloc cap of a client by what its GPU has lent.
 *   which = -1: the GPU this engine computes on;  which = i >= 0: peer i of the configuration.
 */
typedef struct nvs_gpu_account {
	int32_t  tracked;       /* 1: this GPU is in the ledger (0: no ledger / driver without UUIDs)   */
	int32_t  device;        /* CUDA ordinal as this process numbers the GPUs                        */
	uint64_t total_bytes;   /* cuDeviceTotalMem (own GPU only; 0 for peers)                         */
	uint64_t reserve_bytes; /* slice nobody may claim (NVSHARE_GPU_RESERVE_MIB, default 1536 MiB)   */
	uint64_t lent_bytes;    /* backing arenas held on it by processes that compute elsewhere        */
	uint64_t max_own_bytes; /* largest swappable footprint among the processes computing on it      */
	uint64_t my_lent_bytes;
	uint64_t my_own_bytes;
	uint64_t refusals;      /* peer arenas this engine did not create because the GPU had no room   */
} nvs_gpu_account;
int nvs_gpu_account_query(nvs_engine *e, int which, nvs_gpu_account *out);
/* What the GPU this engine computes on has lent to clients of other GPUs (for the hook's cap). */
uint64_t nvs_gpu_lent_bytes(nvs_engine *e);

/* Is dptr the start of an allocation this engine handed out (small pass-through ones included)?
 * 0 = yes (and *req_bytes = the size that was asked for), NVS_E_NOT_OURS = no.  For callers that must
 * decide who frees a pointer before they do anything else with it (cuMemFreeAsync). */
int nvs_lookup(nvs_engine *e, uint64_t dptr, uint64_t *req_bytes);

/* The application is about to write [dptr, dptr+bytes) from the host side of the API (a
 * cuMemcpy* / cuMemset* destination seen by the hook).  Only a hint: chunks touched recently
 * are the last to be chosen by a partial eviction (they are the ones most likely to differ
 * from their retained backing copy).  No reference counterpart. */
int nvs_touch(nvs_engine *e, uint64_t dptr, uint64_t bytes);

/* Raw kernel access (parity tests, roofline).  All addresses must be
 * device-accessible in the engine's context.  *ms = CUDA-event time. */
int nvs_copy_slabs(nvs_engine *e, const nvs_copy_desc *descs, uint32_t n, uint32_t variant,
		   uint32_t grid, float *ms);
/* What the scan kernel reports per slab (nvs_slab_scan in slab_copy.cu). */
typedef struct nvs_scan_out {
	uint64_t value;    /* the slab's first 64-bit word                                  */
	uint64_t is_const; /* 1: every 64-bit word of the slab equals `value`               */
	uint64_t h0, h1;   /* 128-bit content hash (0, 0 when not asked for)                */
} nvs_scan_out;
/* Run the scan/hash kernel over descs[i].src / .bytes; out[n].  descs[i].dst == 0: scan only; with
 * want_hash == 0 the scan may stop at the first 32 KiB tile that differs and reports no hash.
 * descs[i].dst != 0: fused copy + hash, as the background pre-cleaner runs it: [src, src+bytes) is
 * copied to dst in full, and the hash is reported whatever want_hash says and describes the bytes
 * that landed in dst.  src, dst and bytes must be multiples of 16 (else NVS_E_BAD_ARG, nothing
 * launched), bytes > 0. */
int nvs_scan_slabs(nvs_engine *e, const nvs_copy_desc *descs, uint32_t n, int want_hash, nvs_scan_out *out,
		   float *ms);
int nvs_pattern_fill(nvs_engine *e, uint64_t addr, uint64_t n_words, uint64_t first_index, uint64_t seed);
int nvs_pattern_verify(nvs_engine *e, uint64_t addr, uint64_t n_words, uint64_t first_index, uint64_t seed,
		       uint64_t *mismatches);

const char *nvs_strerror(int rc);
const char *nvs_engine_version(void);

#ifdef __cplusplus
}
#endif
#endif /* NVSHARE_ENGINE_H */
