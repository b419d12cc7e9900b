/*
 * engine.c -- the H100 swap engine (host side, plain C on the CUDA driver API).
 *
 * The reference has no such component: its whole data path is one call,
 * real_cuMemAllocManaged() (reference src/hook.c:673), after which NVIDIA's
 * UVM driver migrates pages on GPU faults.  This file is that data path made
 * explicit and H100-shaped:
 *
 *   allocation  cuMemAddressReserve for the application's pointer (stable for
 *               the allocation's life) + cuMemCreate/cuMemMap/cuMemSetAccess
 *               per CHUNK (default 256 MiB = 128 slabs).  VMM calls cost per call,
 *               not per byte (tools/probe.cu section B measures it per
 *               mapping-chunk size).  Copy and accounting granularity stays one SLAB (2 MiB).
 *   backing     tier 1: HBM of peer GPUs (cuMemCreate on the peer, mapped into
 *               this context; striped per chunk; arenas returned as soon as they
 *               are empty; no NCCL).  tier 0: pinned host DRAM -- by default ONE
 *               pool per scheduler shared by all its clients (a /dev/shm file,
 *               1 GiB windows registered per process), else private
 *               cuMemHostAlloc arenas.  Backing is released as soon as a batch
 *               has been fetched back.
 *   evict       resident chunks, least recently fetched first -> nvs_slab_scan
 *               (same-filled slabs are described, not moved) -> descriptors ->
 *               nvs_slab_copy_tma on a side stream, batch b+1 copying while
 *               batch b is unmapped and its HBM released.
 *   fetch       the mirror image with the copy engines (the evicting process is
 *               running its kernel at the same time): wait until a BURST
 *               of HBM is free, map it back to back, copy, splat the
 *               same-filled slabs.
 *
 * Chunk states:  UNBACKED (virtual only; contents undefined like fresh
 * cuMemAlloc memory, nothing to copy) -> RESIDENT <-> SWAPPED.
 *
 * Nothing here falls back to a CPU copy: no driver / no kernel image -> error.
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <dlfcn.h>
#include <errno.h>
#include <inttypes.h>
#include <pthread.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <time.h>
#include <unistd.h>
#include <fcntl.h>
#include <signal.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/statvfs.h>

#include "../../include/nvshare_engine.h"
#include "cuda_min.h"
#include "nvs_log.h"
#include "gpu_ledger.h"
#include "slab_copy_cubin.h" /* generated: nvs_slab_copy_cubin[], nvs_slab_copy_cubin_len */

#define SLAB NVS_SLAB_BYTES
#define MAX_CHUNK_SLABS 256u /* chunk_bytes <= 512 MiB */
#define N_SLOTS 3 /* pipeline depth (batches in flight) */

enum { CH_UNBACKED = 0, CH_RESIDENT = 1, CH_SWAPPED = 2 };
enum { TIER_NONE = 0, TIER_HOST = 1, TIER_PEER0 = 2 /* TIER_PEER0 + peer index */ };

/* ----------------------------------------------------------- driver ---- */

struct drv {
	CUresult (*GetErrorName)(CUresult, const char **);
	CUresult (*CtxGetCurrent)(CUcontext *);
	CUresult (*CtxPushCurrent)(CUcontext);
	CUresult (*CtxPopCurrent)(CUcontext *);
	CUresult (*CtxGetDevice)(CUdevice *);
	CUresult (*CtxSynchronize)(void);
	CUresult (*DeviceGetAttribute)(int *, int, CUdevice);
	CUresult (*DeviceCanAccessPeer)(int *, CUdevice, CUdevice);
	CUresult (*MemGetInfo)(size_t *, size_t *);
	CUresult (*MemAlloc)(CUdeviceptr *, size_t);
	CUresult (*MemFree)(CUdeviceptr);
	CUresult (*MemHostAlloc)(void **, size_t, unsigned);
	CUresult (*MemFreeHost)(void *);
	CUresult (*MemHostGetDevicePointer)(CUdeviceptr *, void *, unsigned);
	CUresult (*MemHostRegister)(void *, size_t, unsigned);
	CUresult (*MemHostUnregister)(void *);
	CUresult (*MemAddressReserve)(CUdeviceptr *, size_t, size_t, CUdeviceptr, unsigned long long);
	CUresult (*MemAddressFree)(CUdeviceptr, size_t);
	CUresult (*MemCreate)(CUmemGenericAllocationHandle *, size_t, const CUmemAllocationProp *,
			      unsigned long long);
	CUresult (*MemRelease)(CUmemGenericAllocationHandle);
	CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
	CUresult (*MemUnmap)(CUdeviceptr, size_t);
	CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc *, size_t);
	CUresult (*MemGetAllocationGranularity)(size_t *, const CUmemAllocationProp *, int);
	CUresult (*MemcpyAsync)(CUdeviceptr, CUdeviceptr, size_t, CUstream);
	CUresult (*MemsetD32Async)(CUdeviceptr, unsigned, size_t, CUstream);
	CUresult (*StreamCreate)(CUstream *, unsigned);
	CUresult (*StreamCreateWithPriority)(CUstream *, unsigned, int);        /* optional */
	CUresult (*CtxGetStreamPriorityRange)(int *, int *);                    /* optional */
	CUresult (*DeviceGetUuid)(uint8_t uuid[16], CUdevice);                  /* optional (gpu ledger) */
	CUresult (*DeviceTotalMem)(size_t *, CUdevice);                         /* optional (gpu ledger) */
	CUresult (*DeviceGetCount)(int *);                                      /* optional (NVSHARE_PEERS=auto) */
	CUresult (*StreamDestroy)(CUstream);
	CUresult (*StreamSynchronize)(CUstream);
	CUresult (*EventCreate)(CUevent *, unsigned);
	CUresult (*EventDestroy)(CUevent);
	CUresult (*EventRecord)(CUevent, CUstream);
	CUresult (*EventSynchronize)(CUevent);
	CUresult (*EventQuery)(CUevent);
	CUresult (*EventElapsedTime)(float *, CUevent, CUevent);
	CUresult (*ModuleLoadData)(CUmodule *, const void *);
	CUresult (*ModuleUnload)(CUmodule);
	CUresult (*ModuleGetFunction)(CUfunction *, CUmodule, const char *);
	CUresult (*FuncSetAttribute)(CUfunction, int, int);
	CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned,
				 unsigned, CUstream, void **, void **);
};

static const struct {
	const char *name;
	size_t off;
} DRV_SYMS[] = {
#define S(field, sym) {sym, offsetof(struct drv, field)}
	S(GetErrorName, "cuGetErrorName"),
	S(CtxGetCurrent, "cuCtxGetCurrent"),
	S(CtxPushCurrent, "cuCtxPushCurrent_v2"),
	S(CtxPopCurrent, "cuCtxPopCurrent_v2"),
	S(CtxGetDevice, "cuCtxGetDevice"),
	S(CtxSynchronize, "cuCtxSynchronize"),
	S(DeviceGetAttribute, "cuDeviceGetAttribute"),
	S(DeviceCanAccessPeer, "cuDeviceCanAccessPeer"),
	S(MemGetInfo, "cuMemGetInfo_v2"),
	S(MemAlloc, "cuMemAlloc_v2"),
	S(MemFree, "cuMemFree_v2"),
	S(MemHostAlloc, "cuMemHostAlloc"),
	S(MemFreeHost, "cuMemFreeHost"),
	S(MemHostGetDevicePointer, "cuMemHostGetDevicePointer_v2"),
	S(MemHostRegister, "cuMemHostRegister_v2"),
	S(MemHostUnregister, "cuMemHostUnregister"),
	S(MemAddressReserve, "cuMemAddressReserve"),
	S(MemAddressFree, "cuMemAddressFree"),
	S(MemCreate, "cuMemCreate"),
	S(MemRelease, "cuMemRelease"),
	S(MemMap, "cuMemMap"),
	S(MemUnmap, "cuMemUnmap"),
	S(MemSetAccess, "cuMemSetAccess"),
	S(MemGetAllocationGranularity, "cuMemGetAllocationGranularity"),
	S(MemcpyAsync, "cuMemcpyAsync"),
	S(MemsetD32Async, "cuMemsetD32Async"),
	S(StreamCreate, "cuStreamCreate"),
	S(StreamDestroy, "cuStreamDestroy_v2"),
	S(StreamSynchronize, "cuStreamSynchronize"),
	S(EventCreate, "cuEventCreate"),
	S(EventDestroy, "cuEventDestroy_v2"),
	S(EventRecord, "cuEventRecord"),
	S(EventSynchronize, "cuEventSynchronize"),
	S(EventQuery, "cuEventQuery"),
	S(EventElapsedTime, "cuEventElapsedTime"),
	S(ModuleLoadData, "cuModuleLoadData"),
	S(ModuleUnload, "cuModuleUnload"),
	S(ModuleGetFunction, "cuModuleGetFunction"),
	S(FuncSetAttribute, "cuFuncSetAttribute"),
	S(LaunchKernel, "cuLaunchKernel"),
#undef S
};

static void *default_resolve(const char *symbol)
{
	static void *lib;
	if (!lib)
		lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
	return lib ? dlsym(lib, symbol) : NULL;
}

/* ------------------------------------------------------------- types ---- */

struct chunk {
	uint64_t va;
	uint64_t bytes;
	CUmemGenericAllocationHandle handle; /* valid while RESIDENT */
	uint64_t backing;                    /* device-accessible address of the backing range, 0 = none */
	uint64_t epoch;                      /* engine epoch at which it last became resident */
	struct alloc *owner;
	uint8_t state;
	uint8_t tier;
	/* same-filled slabs found at eviction: bit i set = slab i is `cvals[i]` repeated,
	 * was not copied out and is re-created by nvs_slab_splat at fetch */
	uint32_t n_const;
	uint64_t cmask[MAX_CHUNK_SLABS / 64];
	uint64_t *cvals;
	/* Clean-slab skip.  `backing` may outlive a fetch (`retained`): the pool keeps the
	 * units marked as reclaimable, anybody short of units may take them over, and the
	 * owner finds out when it validates the run under the pool lock (backing_reclaim).
	 * hash[i] is the content hash of the bytes slab i has in the backing, valid where
	 * bvalid has bit i set; an eviction copies slab i only if its current hash differs. */
	uint8_t retained;   /* RESIDENT with a backing copy that MAY still be ours             */
	uint8_t stable;     /* ST_UNKNOWN / ST_STABLE (found clean last time) / ST_VOLATILE    */
	uint8_t scanned;    /* this eviction has already scanned it: cpmask / nh / cmask valid */
	uint8_t had_backing; /* ... and it went into the scan with a valid backing copy        */
	uint8_t volatile_skips; /* fetches since a volatile chunk's backing was last retained  */
	uint64_t pre_epoch;  /* engine epoch in which the pre-cleaner last looked at this chunk  */
	uint32_t btag;      /* tag written next to our units in the pool: proves they are still ours */
	uint64_t touch;     /* engine touch clock of the last host-side write (nvs_touch)      */
	uint64_t est_copy;  /* bytes this eviction would have to copy (from the scan)          */
	uint64_t bvalid[MAX_CHUNK_SLABS / 64];
	uint64_t cpmask[MAX_CHUNK_SLABS / 64]; /* slabs this eviction must copy               */
	struct slab_hash *hash; /* [MAX_CHUNK_SLABS], lazily allocated                         */
	struct slab_hash *nh;   /* hashes of the current contents, during an eviction only     */
};

struct slab_hash {
	uint64_t h0, h1;
};
enum { ST_UNKNOWN = 0, ST_STABLE = 1, ST_VOLATILE = 2 };
/* a volatile chunk's backing is kept again every so many fetches, to notice that it calmed down */
#define VOLATILE_REPROBE 8

struct alloc {
	uint64_t va;
	uint64_t req_bytes;
	uint64_t va_bytes;
	uint32_t n_chunks;
	int passthrough;
	struct chunk *chunks;
	struct alloc *hnext;       /* hash bucket chain          */
	struct alloc *prev, *next; /* allocation order           */
};

struct arena {
	uint64_t dev_base;  /* device-accessible base address              */
	void *host_base;    /* host tier: pointer to free; NULL for peers  */
	CUmemGenericAllocationHandle handle; /* peer tier                   */
	uint64_t bytes;
	uint32_t n_slabs, used;
	uint32_t hint;      /* private pool: first slab worth scanning     */
	uint64_t *bitmap;   /* 1 = slab in use                             */
	int32_t *owners;    /* shared pool only: pid owning each slab      */
	uint8_t *rstate;    /* per slab: 0 = free or live, RS_* = retained (reclaimable) */
	uint32_t *ctag;     /* per slab: tag of the chunk the unit was handed to         */
	int shared;         /* bitmap/owners/rstate/ctag live in the shared pool header  */
	uint64_t bit_base;  /* index of this arena's slab 0 in `bitmap` / `owners` (shared pool: global) */
	uint32_t window;    /* shared pool only: index of this 1 GiB window */
	struct arena *next;
};

/*
 * Shared pinned-host pool: ONE backing store for every client of a scheduler
 * (a file in /dev/shm mapped by all of them), so that host RAM tracks what is
 * actually swapped out (~0.5 C for two clients at 1.5x) instead of the sum of
 * per-process pools (~1.0-1.5 C).  Where pinned memory is charged to a memory
 * cgroup, the per-process pools of the BASELINE configuration can exceed it.  Layout of the file:
 *   [0, SHP_HDR_BYTES)   struct shp_hdr: robust process-shared mutex, slab
 *                        bitmap, owner pid per slab
 *   [SHP_HDR_BYTES, ..)  data: capacity_slabs x 2 MiB, handed out in contiguous
 *                        runs that never straddle a 1 GiB registration window
 * Each process cuMemHostRegister()s a window the first time it needs it.
 */
#define SHP_MAGIC 0x6e767368504f4f4cull /* "nvshPOOL" */
#define SHP_HDR_BYTES (8ull << 20)
#define SHP_MAX_SLABS (1u << 19) /* 1 TiB */
#define SHP_VERSION 3

struct shp_hdr {
	volatile uint64_t magic;
	uint32_t version;
	uint32_t window_slabs;
	uint64_t capacity_slabs;
	uint64_t used_slabs;
	pthread_mutex_t mu;
	uint64_t bitmap[SHP_MAX_SLABS / 64];
	int32_t owners[SHP_MAX_SLABS];
	uint8_t rstate[SHP_MAX_SLABS]; /* RS_*: the unit holds a copy its owner can do without */
	uint32_t ctag[SHP_MAX_SLABS];
	/* Hand-over progress, written by the client that is evicting for the next holder and read by
	 * the one that is fetching: how much HBM the eviction announced by `releaser_pid` has given
	 * back so far.  The fetching side waits on these words instead of polling cuMemGetInfo every
	 * millisecond -- driver calls of two processes at the moment one of them runs hundreds of
	 * cuMemUnmap / cuMemRelease back to back are exactly what makes the release slow. */
	volatile int32_t releaser_pid;       /* 0: nobody is releasing                           */
	volatile uint32_t release_seq;       /* bumped at every announcement                     */
	volatile uint64_t released_bytes;    /* since the announcement                           */
	/* Owners are identified by pid and their liveness is checked with kill(pid, 0): that only means
	 * something inside ONE pid namespace.  Clients of another one (containers that share /dev/shm
	 * but not the pid namespace) must not attach -- they would reap the units of live owners. */
	uint64_t pid_ns;                     /* inode of the creator's /proc/self/ns/pid, 0 = unknown */
};
enum { RS_NONE = 0, RS_PLAIN = 1, RS_STABLE = 2 }; /* reclaim order: free, then PLAIN, then STABLE */
_Static_assert(sizeof(struct shp_hdr) <= SHP_HDR_BYTES, "shared pool header too large");

struct shpool {
	int fd;
	struct shp_hdr *hdr;
	uint8_t *data;       /* host VA of the data region (whole capacity mapped, registered per window) */
	uint32_t n_windows;
	uint8_t *registered; /* per window: this process has it pinned */
	char path[256];
};

struct pool {
	struct arena *arenas;
	uint64_t bytes, used;
	uint64_t capacity; /* 0 = unlimited */
	int device;        /* peer ordinal, -1 for the host tier */
	int gl_dev;        /* that GPU's index in the cross-process ledger (gpu_ledger.h), -1 = not tracked */
	uint64_t gl_refusals; /* arenas not created because the ledger said that GPU has no room to lend */
};

struct scan_result;
struct slot {
	nvs_copy_desc *descs; /* pinned, device-mapped: what the sm_90a copy kernel consumes */
	uint64_t descs_dev;
	uint32_t n_descs, cap_descs;
	nvs_copy_desc *ce;    /* plain host memory: runs handed to the copy engines            */
	uint32_t n_ce, cap_ce;
	int peer_traffic;     /* the kernel list touches peer HBM: wants the NVLink-sized grid */
	struct chunk **chunks;
	uint32_t n_chunks, cap_chunks;
	CUevent begin, done; /* around this batch's copy: device time of the copy alone */
	int busy;
	/* auxiliary descriptor list: scan inputs (evict) or splat list (fetch), and scan results */
	nvs_copy_desc *aux;
	uint64_t aux_dev;
	uint32_t n_aux, cap_aux;
	struct scan_result *scan_out;
	uint64_t scan_out_dev;
};

struct scan_result {
	uint64_t value;
	uint64_t is_const;
	uint64_t h0, h1;
};
_Static_assert(sizeof(struct scan_result) == sizeof(nvs_scan_out), "scan result layout is part of the C-ABI");

#define HASH_BITS 12
#define HASH_SIZE (1u << HASH_BITS)

struct nvs_engine {
	struct drv d;
	nvs_engine_config cfg;
	CUcontext ctx;
	int device;
	int n_sms;
	CUmodule module;
	CUfunction fn_tma, fn_ldg, fn_fill, fn_verify, fn_scan, fn_splat;
	CUstream stream;
	CUstream scan_stream; /* the scan of batch b+1 runs beside the copy of batch b */
	CUevent scan_done, scan_begin;
	uint32_t scan_counter_next;
	uint64_t touch_clock;
	uint32_t tag_next;
	/* background pre-cleaning (preclean_main) */
	pthread_t pre_thread;
	int pre_thread_started;
	pthread_cond_t pre_cv;
	CUstream pre_stream; /* lowest priority: never in the way of the application's kernels */
	CUevent pre_done;
	nvs_copy_desc *pre_descs;
	uint64_t pre_descs_dev;
	struct scan_result *pre_out;
	uint64_t pre_out_dev;
	CUdeviceptr pre_counter;
	CUevent ev_begin, ev_end;
	CUdeviceptr counters; /* u32[N_COUNTERS], device memory */
	uint32_t counter_next;
	CUdeviceptr scratch;  /* u64 mismatch counter           */
	struct slot slots[N_SLOTS];

	pthread_mutex_t api_mu; /* outer: serialises the public entry points                   */
	pthread_mutex_t mu;     /* inner: table, pools, stats (shared with the pinning thread) */
	struct alloc *buckets[HASH_SIZE];
	struct alloc *head, *tail;
	struct alloc **by_va; /* every allocation, sorted by address: range lookups in O(log n) */
	size_t n_by_va, cap_by_va;
	struct pool host_pool;
	struct shpool *shp; /* non-NULL: host_pool's arenas are windows of the shared pool */
	struct pool peer_pools[NVS_MAX_PEERS];
	uint32_t peer_rr;
	int gl_dev;          /* the GPU we compute on, in the cross-process ledger (-1 = not tracked) */
	uint64_t gl_reserve; /* bytes of every GPU that are nobody's to claim (contexts, libraries)  */
	uint64_t gl_total;   /* cuDeviceTotalMem of the GPU we compute on                            */
	uint64_t epoch;
	int resident_mode;
	nvs_stats st;

	/* background pinning */
	pthread_t pin_thread;
	int pin_thread_started;
	pthread_cond_t pin_cv;
	pthread_cond_t grow_cv; /* an arena finished pinning (or failed) */
	int growing;            /* a thread is inside cuMemHostAlloc for a new arena */
	int stopping;
	uint64_t pin_target; /* bytes of host pool we want to have */

	FILE *stats_file;

	/* CPUs on the GPU's own NUMA node: threads that first-touch (i.e. place) pinned
	 * backing pages run there, so that the DMA does not cross the socket interconnect */
	cpu_set_t near_cpus;
	int near_cpus_valid;
	double pool_grace_ms; /* POOL_FULL_GRACE_MS, or NVSHARE_POOL_GRACE_MS */
};
#define N_COUNTERS 1024u /* per stream; the scan stream uses the second half of the array */
/* Memory pressure is only signalled once the free HBM has not grown for this long: while
 * the previous holder is evicting for us it grows every few tens of ms, and a pressure
 * message sent then would be handled AFTER that eviction and evict the same amount again. */
#define PRESSURE_AFTER_MS 300.0
/* how long an eviction waits for units of a full shared pool before it pins an overflow arena */
#define POOL_FULL_GRACE_MS 2000.0

static double now_ms(void)
{
	struct timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

static double wall_s(void)
{
	struct timespec ts;
	clock_gettime(CLOCK_REALTIME, &ts);
	return ts.tv_sec + ts.tv_nsec * 1e-9;
}

static const char *cu_name(nvs_engine *e, CUresult r)
{
	const char *n = NULL;
	if (e->d.GetErrorName && e->d.GetErrorName(r, &n) == CUDA_SUCCESS && n)
		return n;
	return "CUDA_ERROR_?";
}

/* The driver is going away under us (the application is exiting and its context
 * has been or is being destroyed): not an engine failure. */
static int is_shutdown_error(CUresult r)
{
	return r == 4 /* DEINITIALIZED */ || r == CUDA_ERROR_NOT_INITIALIZED || r == CUDA_ERROR_INVALID_CONTEXT ||
	       r == 709 /* CONTEXT_IS_DESTROYED */;
}

#define CK(e, call)                                                                        \
	do {                                                                               \
		CUresult r_ = (call);                                                      \
		if (r_ != CUDA_SUCCESS) {                                                  \
			if (is_shutdown_error(r_)) {                                       \
				rc = NVS_E_SHUTDOWN;                                       \
			} else {                                                           \
				nvs_warn("engine: %s returned %s (%d) at %s:%d", #call,    \
					 cu_name(e, r_), (int)r_, __FILE__, __LINE__);     \
				rc = (int)r_;                                              \
			}                                                                  \
			goto out;                                                          \
		}                                                                          \
	} while (0)

const char *nvs_engine_version(void)
{
	return "nvshare_b200 engine r2 (sm_90a: slab copy tma|ldg, scan+hash, splat; copy engines for the PCIe tier)";
}

const char *nvs_strerror(int rc)
{
	switch (rc) {
	case 0: return "success";
	case NVS_E_NOT_OURS: return "pointer not owned by the engine";
	case NVS_E_BAD_ARG: return "bad argument";
	case NVS_E_NO_DRIVER: return "CUDA driver (libcuda.so.1) or a required entry point is missing";
	case NVS_E_NO_KERNEL: return "embedded sm_90a kernel image failed to load";
	case NVS_E_TIMEOUT: return "timed out waiting for HBM to be released";
	case NVS_E_HOST_OOM: return "backing tier exhausted";
	case NVS_E_SHUTDOWN: return "the CUDA context is being torn down (process exit)";
	case NVS_E_NOT_SWAPPED: return "the range is (partly) resident on a GPU: use the device path";
	case CUDA_ERROR_OUT_OF_MEMORY: return "CUDA_ERROR_OUT_OF_MEMORY";
	case CUDA_ERROR_NOT_INITIALIZED: return "CUDA_ERROR_NOT_INITIALIZED";
	default: return rc > 0 ? "CUDA driver error" : "unknown engine error";
	}
}

/* ------------------------------------------------------------ config ---- */

static uint64_t env_u64(const char *name, uint64_t dflt)
{
	const char *v = getenv(name);
	if (!v || !*v)
		return dflt;
	char *end = NULL;
	unsigned long long x = strtoull(v, &end, 0);
	return end == v ? dflt : (uint64_t)x;
}

static uint32_t parse_variant(const char *v, uint32_t dflt)
{
	if (!v || !*v)
		return dflt;
	if (!strcasecmp(v, "tma"))
		return NVS_COPY_TMA;
	if (!strcasecmp(v, "ldg"))
		return NVS_COPY_LDG;
	if (!strcasecmp(v, "ce"))
		return NVS_COPY_CE;
	return dflt;
}

int nvs_engine_default_config(nvs_engine_config *cfg)
{
	if (!cfg)
		return NVS_E_BAD_ARG;
	memset(cfg, 0, sizeof(*cfg));
	cfg->struct_size = sizeof(*cfg);
	cfg->device = -1;
	cfg->chunk_bytes = env_u64("NVSHARE_CHUNK_MIB", 256) << 20;
	cfg->small_alloc_bytes = env_u64("NVSHARE_SMALL_ALLOC_KIB", 1024) << 10;
	cfg->batch_bytes = env_u64("NVSHARE_BATCH_MIB", 1024) << 20;
	cfg->burst_bytes = env_u64("NVSHARE_BURST_MIB", 65536) << 20;
	cfg->host_arena_bytes = env_u64("NVSHARE_HOST_ARENA_MIB", 1024) << 20;
	/* Pinned-host tier (PCIe Gen5 x16): the copy engines carry 256-byte TLPs, SM-issued transfers
	 * 128-byte ones, and the copy kernel, being compute work, is time-sliced against the other
	 * process's kernel.  So both directions of this tier run on the copy engines; the SMs scan,
	 * hash and splat.  Peer tier (NVLink): the kernel, which keeps many more bytes in flight than
	 * per-chunk cuMemcpyAsync calls, for both directions.
	 * NVSHARE_COPY_VARIANT sets all four; the specific variables override it. */
	const char *all = getenv("NVSHARE_COPY_VARIANT");
	cfg->evict_variant = parse_variant(getenv("NVSHARE_EVICT_VARIANT"), parse_variant(all, NVS_COPY_CE));
	cfg->fetch_variant = parse_variant(getenv("NVSHARE_FETCH_VARIANT"), parse_variant(all, NVS_COPY_CE));
	cfg->peer_evict_variant = parse_variant(getenv("NVSHARE_PEER_EVICT_VARIANT"), parse_variant(all, NVS_COPY_TMA));
	/* ... except that a FETCH usually runs while the previous holder's eviction kernel is still going
	 * in another process, and the GPU time-slices kernels of different processes: eviction kernel + fetch on the copy
	 * engines overlap, two kernels take turns.  NVSHARE_PEER_FETCH_VARIANT=tma for a fetch that has
	 * the GPU to itself. */
	cfg->peer_fetch_variant = parse_variant(getenv("NVSHARE_PEER_FETCH_VARIANT"), parse_variant(all, NVS_COPY_CE));
	cfg->retain = (uint32_t)env_u64("NVSHARE_RETAIN", 1);
	cfg->preclean = (uint32_t)env_u64("NVSHARE_PRECLEAN", 1);
	/* 0 = derived per launch (grid_for()): 8 CTAs for the PCIe tier, with head-room for SMs that
	 * are shared with a client's kernels, and half the SMs for the peer tier. */
	cfg->copy_grid = (uint32_t)env_u64("NVSHARE_COPY_GRID", 0);
	cfg->tma_warps = (uint32_t)env_u64("NVSHARE_TMA_WARPS", 1);
	cfg->tma_stages = (uint32_t)env_u64("NVSHARE_TMA_STAGES", 6);
	cfg->tma_tile_bytes = (uint32_t)env_u64("NVSHARE_TMA_TILE_KIB", 32) << 10;
	cfg->ldg_threads = (uint32_t)env_u64("NVSHARE_LDG_THREADS", 512);
	cfg->oom_wait_ms = (uint32_t)env_u64("NVSHARE_OOM_WAIT_MS", 120000);
	cfg->prepin = (uint32_t)env_u64("NVSHARE_PREPIN", 1);
	cfg->peer_capacity_bytes = env_u64("NVSHARE_PEER_CAPACITY_MIB", 0) << 20;
	cfg->elide_constant = (uint32_t)env_u64("NVSHARE_ELIDE", 1);
	cfg->stats_path = getenv("NVSHARE_STATS_FILE");
	cfg->shared_pool_path = getenv("NVSHARE_POOL_PATH"); /* libnvshare.so derives one from the socket path */
	cfg->shared_pool_bytes = env_u64("NVSHARE_POOL_GIB", 0) << 30;
	if (getenv("NVSHARE_POOL_MIB")) /* finer grain, for tests of a tight pool */
		cfg->shared_pool_bytes = env_u64("NVSHARE_POOL_MIB", 0) << 20;
	const char *peers = getenv("NVSHARE_PEERS"); /* "1,2,3", or "auto" */
	if (peers && !strcmp(peers, "auto")) {
		cfg->n_peers = NVS_PEERS_AUTO;
	} else if (peers && *peers) {
		char buf[128];
		snprintf(buf, sizeof(buf), "%s", peers);
		char *save = NULL; /* strtok_r: this library lives inside arbitrary applications */
		for (char *tok = strtok_r(buf, ",", &save); tok && cfg->n_peers < NVS_MAX_PEERS; tok = strtok_r(NULL, ",", &save))
			cfg->peers[cfg->n_peers++] = atoi(tok);
	}
	return 0;
}

/* --------------------------------------------------------- ctx guard ---- */

static int ctx_enter(nvs_engine *e)
{
	return e->d.CtxPushCurrent(e->ctx) == CUDA_SUCCESS ? 0 : -1;
}
/* entry points return this when the context cannot be entered: at process exit
 * that is normal, so it is reported as a shutdown, not as a failure */
#define CTX_GONE NVS_E_SHUTDOWN

static void ctx_leave(nvs_engine *e)
{
	CUcontext junk;
	e->d.CtxPopCurrent(&junk);
}

/* -------------------------------------------------------------- NUMA ---- */

/* "0-3,8,10-11" -> cpu_set_t; returns the number of CPUs */
static int parse_cpulist(const char *s, cpu_set_t *set)
{
	CPU_ZERO(set);
	int n = 0;
	while (*s) {
		char *end;
		long a = strtol(s, &end, 10), b = a;
		if (end == s)
			break;
		if (*end == '-') {
			s = end + 1;
			b = strtol(s, &end, 10);
			if (end == s)
				break;
		}
		for (long c = a; c <= b && c >= 0 && c < CPU_SETSIZE; ++c) {
			CPU_SET((int)c, set);
			n++;
		}
		s = *end == ',' ? end + 1 : end;
		if (*end != ',')
			break;
	}
	return n;
}

/*
 * Where should pinned backing memory live?  On a two-socket host the GPU hangs off
 * one socket; pages first-touched by a thread on the other one are reached by every
 * DMA through the socket interconnect.  Linux places a page on the node of the CPU
 * that faults it in, so the threads that populate the pool are confined to the
 * GPU's local CPUs (sysfs local_cpulist of its PCI function) while they do so --
 * sched_setaffinity needs no privilege, unlike mbind under the usual container
 * seccomp profile.  NVSHARE_NUMA=1 turns it on; NVSHARE_NUMA_CPULIST overrides sysfs.
 */
static void numa_init(nvs_engine *e, CUdevice dev, nvs_resolve_fn resolve)
{
	/* Opt-in (NVSHARE_NUMA=1): on a two-socket box the socket interconnect is not the bottleneck of
	 * a PCIe transfer, so the default leaves the pages where the kernel puts them. */
	const char *sw = getenv("NVSHARE_NUMA");
	if (!(sw && *sw && atoi(sw) != 0))
		return;
	char list[512] = "";
	const char *forced = getenv("NVSHARE_NUMA_CPULIST");
	if (forced && *forced) {
		snprintf(list, sizeof(list), "%s", forced);
	} else {
		CUresult (*get_bus_id)(char *, int, CUdevice) = (CUresult (*)(char *, int, CUdevice))resolve("cuDeviceGetPCIBusId");
		char bdf[64] = "", path[160];
		if (!get_bus_id || get_bus_id(bdf, (int)sizeof(bdf) - 1, dev) != CUDA_SUCCESS || !bdf[0])
			return;
		for (char *c = bdf; *c; ++c)
			if (*c >= 'A' && *c <= 'F')
				*c = (char)(*c - 'A' + 'a');
		snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", bdf);
		FILE *f = fopen(path, "r");
		if (!f)
			return;
		if (!fgets(list, sizeof(list), f))
			list[0] = '\0';
		fclose(f);
	}
	cpu_set_t want, allowed;
	if (parse_cpulist(list, &want) == 0 || sched_getaffinity(0, sizeof(allowed), &allowed) != 0)
		return;
	CPU_AND(&e->near_cpus, &want, &allowed);
	const int n_near = CPU_COUNT(&e->near_cpus), n_allowed = CPU_COUNT(&allowed);
	if (n_near == 0 || n_near == n_allowed)
		return; /* nothing to choose from, or a single node: leave the threads alone */
	e->near_cpus_valid = 1;
	nvs_debug("engine: pinned backing memory is placed from %d of %d CPUs (the GPU's NUMA node)", n_near, n_allowed);
}

/* confine the calling thread to the GPU's CPUs; returns 1 if *saved must be restored */
static int near_push(nvs_engine *e, cpu_set_t *saved)
{
	if (!e->near_cpus_valid || pthread_getaffinity_np(pthread_self(), sizeof(*saved), saved) != 0)
		return 0;
	return pthread_setaffinity_np(pthread_self(), sizeof(e->near_cpus), &e->near_cpus) == 0;
}

static void near_pop(int pushed, const cpu_set_t *saved)
{
	if (pushed)
		pthread_setaffinity_np(pthread_self(), sizeof(*saved), saved);
}

/* -------------------------------------------------------------- pool ---- */

static inline int bit_get(const struct arena *a, uint32_t i)
{
	uint64_t k = a->bit_base + i;
	return (a->bitmap[k >> 6] >> (k & 63)) & 1;
}

static inline void bit_put(struct arena *a, uint32_t i, int v, int32_t owner, uint32_t tag)
{
	uint64_t k = a->bit_base + i;
	if (v)
		a->bitmap[k >> 6] |= 1ull << (k & 63);
	else
		a->bitmap[k >> 6] &= ~(1ull << (k & 63));
	if (a->owners)
		a->owners[k] = owner;
	a->rstate[k] = RS_NONE;
	a->ctag[k] = tag;
}

/* may slab i be handed out?  free always; a retained unit if its class is <= steal_class */
static inline int slab_available(const struct arena *a, uint32_t i, int steal_class)
{
	if (!bit_get(a, i))
		return 1;
	const uint8_t rs = a->rstate[a->bit_base + i];
	return rs != RS_NONE && (int)rs <= steal_class;
}

/*
 * First fit of n adjacent units (runs never straddle arenas).  steal_class 0 takes free
 * units only; 1 / 2 also take over retained units (RS_PLAIN / RS_STABLE) -- copies their
 * owners can do without, whoever they are.  The owner notices through the tag
 * (backing_reclaim).  *fresh = how many of the n units were free before.
 */
static int arena_take(struct arena *a, uint32_t n, uint64_t *addr, int steal_class, uint32_t tag, uint32_t *fresh)
{
	if (!a->shared && steal_class == 0 && a->n_slabs - a->used < n)
		return -1;
	uint32_t run = 0;
	for (uint32_t i = (a->shared || steal_class) ? 0 : a->hint; i < a->n_slabs; ++i) {
		/* 64 units in use at a stroke (the common case in a busy pool) */
		if (steal_class == 0 && ((a->bit_base + i) & 63) == 0 && i + 64 <= a->n_slabs &&
		    a->bitmap[(a->bit_base + i) >> 6] == ~0ull) {
			run = 0;
			i += 63;
			continue;
		}
		if (!slab_available(a, i, steal_class)) {
			run = 0;
			continue;
		}
		if (++run == n) {
			uint32_t first = i + 1 - n, was_free = 0;
			for (uint32_t k = first; k <= i; ++k) {
				was_free += !bit_get(a, k);
				bit_put(a, k, 1, (int32_t)getpid(), tag);
			}
			a->used += was_free;
			while (!a->shared && a->hint < a->n_slabs && bit_get(a, a->hint))
				a->hint++;
			*addr = a->dev_base + (uint64_t)first * SLAB;
			*fresh = was_free;
			return 0;
		}
	}
	return -1;
}

/* the shared pool's mutex is robust: a client that dies holding it does not wedge the others */
static void shp_lock(struct shpool *sp)
{
	int rc = pthread_mutex_lock(&sp->hdr->mu);
	if (rc == EOWNERDEAD)
		pthread_mutex_consistent(&sp->hdr->mu);
}

static void shp_unlock(struct shpool *sp)
{
	pthread_mutex_unlock(&sp->hdr->mu);
}

static int pool_take(nvs_engine *e, struct pool *p, uint32_t n, uint64_t *addr, int steal_class, uint32_t tag)
{
	struct shpool *sp = (p == &e->host_pool) ? e->shp : NULL;
	int rc = -1;
	if (sp)
		shp_lock(sp);
	for (struct arena *a = p->arenas; a; a = a->next) {
		uint32_t fresh = 0;
		if (arena_take(a, n, addr, steal_class, tag, &fresh) == 0) {
			p->used += (uint64_t)fresh * SLAB;
			if (sp && a->shared)
				sp->hdr->used_slabs += fresh;
			e->st.stolen_slabs_total += n - fresh;
			rc = 0;
			break;
		}
	}
	if (sp)
		shp_unlock(sp);
	return rc;
}

static struct arena *arena_of(struct pool *p, uint64_t addr)
{
	for (struct arena *a = p->arenas; a; a = a->next)
		if (addr >= a->dev_base && addr < a->dev_base + a->bytes)
			return a;
	return NULL;
}

/* Hand back the units of a run that are (still) ours: tag and, in the shared pool, pid match. */
static void pool_give(nvs_engine *e, struct pool *p, uint64_t addr, uint32_t n, uint32_t tag)
{
	struct shpool *sp = (p == &e->host_pool) ? e->shp : NULL;
	if (sp)
		shp_lock(sp);
	struct arena *a = arena_of(p, addr);
	if (a) {
		const uint32_t first = (uint32_t)((addr - a->dev_base) / SLAB);
		uint32_t given = 0;
		for (uint32_t k = first; k < first + n; ++k) {
			const uint64_t g = a->bit_base + k;
			if (!bit_get(a, k) || a->ctag[g] != tag || (a->owners && a->owners[g] != (int32_t)getpid()))
				continue; /* taken over by somebody else meanwhile */
			bit_put(a, k, 0, 0, 0);
			given++;
		}
		a->used -= given;
		if (!a->shared && first < a->hint)
			a->hint = first;
		p->used -= (uint64_t)given * SLAB;
		if (sp && a->shared)
			sp->hdr->used_slabs -= given;
	}
	if (sp)
		shp_unlock(sp);
}

/* The chunk has been fetched: its units stay, marked as reclaimable by anybody. */
static void pool_mark_retained(nvs_engine *e, struct pool *p, uint64_t addr, uint32_t n, uint8_t rs)
{
	struct shpool *sp = (p == &e->host_pool) ? e->shp : NULL;
	if (sp)
		shp_lock(sp);
	struct arena *a = arena_of(p, addr);
	if (a) {
		const uint32_t first = (uint32_t)((addr - a->dev_base) / SLAB);
		for (uint32_t k = first; k < first + n; ++k)
			a->rstate[a->bit_base + k] = rs;
	}
	if (sp)
		shp_unlock(sp);
}

/* Is the retained run still entirely ours?  Yes: it becomes live again (nobody can take it
 * over any more), returns 1.  No: what is left of it is given back, returns 0. */
static int pool_reclaim(nvs_engine *e, struct pool *p, uint64_t addr, uint32_t n, uint32_t tag)
{
	struct shpool *sp = (p == &e->host_pool) ? e->shp : NULL;
	int ok = 0;
	if (sp)
		shp_lock(sp);
	struct arena *a = arena_of(p, addr);
	if (a) {
		const uint32_t first = (uint32_t)((addr - a->dev_base) / SLAB);
		ok = 1;
		for (uint32_t k = first; k < first + n && ok; ++k) {
			const uint64_t g = a->bit_base + k;
			ok = bit_get(a, k) && a->ctag[g] == tag && a->rstate[g] != RS_NONE &&
			     (!a->owners || a->owners[g] == (int32_t)getpid());
		}
		if (ok)
			for (uint32_t k = first; k < first + n; ++k)
				a->rstate[a->bit_base + k] = RS_NONE;
	}
	if (sp)
		shp_unlock(sp);
	if (!ok)
		pool_give(e, p, addr, n, tag);
	return ok;
}

/* a private arena's own bookkeeping (a shared window's lives in the pool header) */
static void arena_free(struct arena *a)
{
	if (!a->shared) {
		free(a->bitmap);
		free(a->rstate);
		free(a->ctag);
	}
	free(a);
}

static struct arena *arena_new(uint64_t bytes)
{
	struct arena *a = calloc(1, sizeof(*a));
	if (!a)
		return NULL;
	a->bytes = bytes;
	a->n_slabs = (uint32_t)(bytes / SLAB);
	a->bitmap = calloc((a->n_slabs + 63) / 64, sizeof(uint64_t));
	a->rstate = calloc(a->n_slabs ? a->n_slabs : 1, 1);
	a->ctag = calloc(a->n_slabs ? a->n_slabs : 1, sizeof(uint32_t));
	if (!a->bitmap || !a->rstate || !a->ctag) {
		arena_free(a);
		return NULL;
	}
	return a;
}

struct touch_job {
	volatile const uint8_t *p;
	size_t bytes;
	nvs_engine *e;
};

static void *touch_worker(void *arg)
{
	/* READ faults only: the pages may already hold another client's evicted data */
	struct touch_job *j = arg;
	cpu_set_t saved;
	near_push(j->e, &saved); /* this thread ends here: nothing to restore */
	uint8_t acc = 0;
	for (size_t off = 0; off < j->bytes; off += 4096)
		acc ^= j->p[off];
	return (void *)(uintptr_t)acc;
}

/* Which NUMA nodes hold the pool's pages (whole mapping, from /proc/self/numa_maps): evidence for numa_init */
static void report_placement(nvs_engine *e, struct shpool *sp, uint32_t window)
{
	FILE *f = fopen("/proc/self/numa_maps", "r");
	if (!f)
		return;
	char want[32], *line = NULL;
	size_t cap = 0;
	snprintf(want, sizeof(want), "%lx ", (unsigned long)(uintptr_t)sp->hdr);
	while (getline(&line, &cap, f) > 0) {
		if (strncmp(line, want, strlen(want)) != 0)
			continue;
		unsigned long long pages[8] = {0};
		char *save = NULL;
		for (char *t = strtok_r(line, " \n", &save); t; t = strtok_r(NULL, " \n", &save)) {
			unsigned node;
			unsigned long long n;
			if (sscanf(t, "N%u=%llu", &node, &n) == 2 && node < 8)
				pages[node] = n;
		}
		nvs_debug("engine: shared pool window %u pinned; pages per NUMA node: N0=%llu N1=%llu N2=%llu N3=%llu", window,
			  pages[0], pages[1], pages[2], pages[3]);
		if (e->stats_file) {
			fprintf(e->stats_file, "{\"op\":\"pin\",\"t\":%.6f,\"pid\":%d,\"window\":%u,\"near_cpus\":%d,"
				"\"pages_per_node\":[%llu,%llu,%llu,%llu]}\n", wall_s(), (int)getpid(), window,
				e->near_cpus_valid ? CPU_COUNT(&e->near_cpus) : 0, pages[0], pages[1], pages[2], pages[3]);
			fflush(e->stats_file);
		}
		break;
	}
	free(line);
	fclose(f);
}

/* Pin the next window of the shared pool into this process.  e->mu NOT held. */
static int shared_pool_grow_unlocked(nvs_engine *e)
{
	struct shpool *sp = e->shp;
	uint32_t w;
	for (w = 0; w < sp->n_windows && sp->registered[w]; ++w)
		;
	if (w == sp->n_windows)
		return NVS_E_HOST_OOM; /* every window is pinned here already: the pool itself is full */
	const uint64_t win_bytes = (uint64_t)sp->hdr->window_slabs * SLAB;
	uint8_t *base = sp->data + (uint64_t)w * win_bytes;
	/* populate the page cache in parallel (page faults scale across cores; a lone
	 * cuMemHostRegister would fault the pages in one by one) */
	enum { NT = 8 };
	pthread_t th[NT];
	struct touch_job jobs[NT];
	int started = 0;
	for (int i = 0; i < NT; ++i) {
		jobs[i].p = base + (win_bytes / NT) * (uint64_t)i;
		jobs[i].bytes = win_bytes / NT;
		jobs[i].e = e;
		if (pthread_create(&th[i], NULL, touch_worker, &jobs[i]) != 0)
			break;
		started++;
	}
	for (int i = 0; i < started; ++i)
		pthread_join(th[i], NULL);
	cpu_set_t saved;
	const int pushed = near_push(e, &saved); /* pages the workers left to the driver are placed from here */
	CUresult r = e->d.MemHostRegister(base, win_bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP);
	near_pop(pushed, &saved);
	if (r != CUDA_SUCCESS) {
		nvs_warn("engine: cuMemHostRegister of shared pool window %u failed: %s", w, cu_name(e, r));
		return NVS_E_HOST_OOM;
	}
	CUdeviceptr dp = 0;
	if (e->d.MemHostGetDevicePointer(&dp, base, 0) != CUDA_SUCCESS)
		dp = (CUdeviceptr)(uintptr_t)base;
	/* (walking numa_maps costs ~1 s once the mapping holds 100+ GB: never on every window) */
	if (e->near_cpus_valid && (e->stats_file || nvs_debug_enabled) && (sp->n_windows <= 8 || (w + 1) % 32 == 0))
		report_placement(e, sp, w);
	struct arena *a = calloc(1, sizeof(*a));
	if (!a)
		return NVS_E_HOST_OOM;
	a->shared = 1;
	a->window = w;
	a->bytes = win_bytes;
	a->n_slabs = sp->hdr->window_slabs;
	a->bitmap = sp->hdr->bitmap;
	a->owners = sp->hdr->owners;
	a->rstate = sp->hdr->rstate;
	a->ctag = sp->hdr->ctag;
	a->bit_base = (uint64_t)w * sp->hdr->window_slabs;
	a->host_base = base;
	a->dev_base = dp;
	pthread_mutex_lock(&e->mu);
	sp->registered[w] = 1;
	/* keep the list in window order so that first-fit packs the low end of the file */
	struct arena **pp = &e->host_pool.arenas;
	while (*pp && (*pp)->window < w)
		pp = &(*pp)->next;
	a->next = *pp;
	*pp = a;
	e->host_pool.bytes += a->bytes;
	e->st.host_pool_bytes = e->host_pool.bytes;
	pthread_mutex_unlock(&e->mu);
	return 0;
}

/* The slow part: cuMemHostAlloc of one arena.  e->mu NOT held; ctx must be current. */
static int host_pool_grow_unlocked(nvs_engine *e)
{
	if (e->shp)
		return shared_pool_grow_unlocked(e);
	struct arena *a = arena_new(e->cfg.host_arena_bytes);
	if (!a)
		return NVS_E_HOST_OOM;
	void *p = NULL;
	cpu_set_t saved;
	const int pushed = near_push(e, &saved); /* the driver populates the pages from this thread */
	CUresult r = e->d.MemHostAlloc(&p, a->bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP);
	near_pop(pushed, &saved);
	if (r != CUDA_SUCCESS) {
		nvs_warn("engine: cuMemHostAlloc(%" PRIu64 " MiB) failed: %s", a->bytes >> 20, cu_name(e, r));
		arena_free(a);
		return NVS_E_HOST_OOM;
	}
	CUdeviceptr dp = 0;
	if (e->d.MemHostGetDevicePointer(&dp, p, 0) != CUDA_SUCCESS)
		dp = (CUdeviceptr)(uintptr_t)p; /* UVA: identical */
	a->host_base = p;
	a->dev_base = dp;
	pthread_mutex_lock(&e->mu);
	a->next = e->host_pool.arenas;
	e->host_pool.arenas = a;
	e->host_pool.bytes += a->bytes;
	e->st.host_pool_bytes = e->host_pool.bytes;
	pthread_mutex_unlock(&e->mu);
	return 0;
}

/* Pin one more host arena.  Called WITH e->mu held; drops it while pinning
 * (slow, ~3.8 GB/s) with `growing` set so that only one thread pins at a time
 * and others wait for the result instead of pinning a second arena. */
static int host_pool_grow(nvs_engine *e)
{
	if (e->growing) {
		pthread_cond_wait(&e->grow_cv, &e->mu);
		return 0; /* the caller re-checks the pool */
	}
	e->growing = 1;
	pthread_mutex_unlock(&e->mu);
	int rc = host_pool_grow_unlocked(e);
	pthread_mutex_lock(&e->mu);
	e->growing = 0;
	pthread_cond_broadcast(&e->grow_cv);
	return rc;
}
/*
 * The shared pool is full and nobody has returned a unit for a while: rather than fail the
 * hand-off, pin a private arena beside it.  (The pool's capacity is a budget for the common
 * case -- one HBM covers any two clients -- not a reason to kill a third large client.)
 * Called with e->mu held; drops it while pinning.  The arena goes to the END of the list, so
 * the shared windows stay preferred, and is kept for reuse until the engine goes away.
 */
static int host_pool_overflow(nvs_engine *e)
{
	struct arena *a = arena_new(e->cfg.host_arena_bytes);
	if (!a)
		return NVS_E_HOST_OOM;
	pthread_mutex_unlock(&e->mu);
	void *p = NULL;
	cpu_set_t saved;
	const int pushed = near_push(e, &saved);
	CUresult r = e->d.MemHostAlloc(&p, a->bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP);
	near_pop(pushed, &saved);
	CUdeviceptr dp = 0;
	if (r == CUDA_SUCCESS && e->d.MemHostGetDevicePointer(&dp, p, 0) != CUDA_SUCCESS)
		dp = (CUdeviceptr)(uintptr_t)p;
	pthread_mutex_lock(&e->mu);
	if (r != CUDA_SUCCESS) {
		nvs_warn("engine: the shared pool is full and cuMemHostAlloc(%" PRIu64 " MiB) for an overflow arena failed: %s",
			 a->bytes >> 20, cu_name(e, r));
		arena_free(a);
		return NVS_E_HOST_OOM;
	}
	a->host_base = p;
	a->dev_base = dp;
	a->window = UINT32_MAX;
	struct arena **pp = &e->host_pool.arenas;
	while (*pp)
		pp = &(*pp)->next;
	*pp = a;
	e->host_pool.bytes += a->bytes;
	e->st.host_pool_bytes = e->host_pool.bytes;
	nvs_debug("engine: shared pool full; pinned a private overflow arena of %" PRIu64 " MiB", a->bytes >> 20);
	return 0;
}

/* Put GPU `ordinal` (as this process numbers them) into the cross-process ledger: by UUID, because
 * CUDA_VISIBLE_DEVICES renumbers the GPUs per process.  -1: not tracked (no ledger, or a driver
 * without the two queries). */
static int gl_register(nvs_engine *e, int ordinal, uint64_t *total_out)
{
	uint8_t uuid[16];
	size_t total = 0;
	if (total_out)
		*total_out = 0;
	if (!e->d.DeviceGetUuid || !e->d.DeviceTotalMem || e->d.DeviceGetUuid(uuid, (CUdevice)ordinal) != CUDA_SUCCESS ||
	    e->d.DeviceTotalMem(&total, (CUdevice)ordinal) != CUDA_SUCCESS)
		return -1;
	if (total_out)
		*total_out = total;
	return nvs_gl_device(uuid, total);
}

int nvs_gpu_account_query(nvs_engine *e, int which, nvs_gpu_account *out)
{
	if (!e || !out || which < -1 || which >= e->cfg.n_peers)
		return NVS_E_BAD_ARG;
	memset(out, 0, sizeof(*out));
	const int gl = which < 0 ? e->gl_dev : e->peer_pools[which].gl_dev;
	out->device = which < 0 ? e->device : e->peer_pools[which].device;
	out->tracked = gl >= 0;
	out->reserve_bytes = e->gl_reserve;
	if (which < 0)
		out->total_bytes = e->gl_total;
	out->lent_bytes = nvs_gl_lent(gl);
	out->max_own_bytes = nvs_gl_max_own(gl);
	out->my_lent_bytes = nvs_gl_mine(gl, NVS_GL_LENT);
	out->my_own_bytes = nvs_gl_mine(gl, NVS_GL_OWN);
	if (which >= 0) {
		pthread_mutex_lock(&e->mu);
		out->refusals = e->peer_pools[which].gl_refusals;
		pthread_mutex_unlock(&e->mu);
	}
	return 0;
}

uint64_t nvs_gpu_lent_bytes(nvs_engine *e)
{
	return e ? nvs_gl_lent(e->gl_dev) : 0;
}

/* Create one arena of peer HBM mapped into this context.  Called with e->mu held. */
static int peer_pool_grow(nvs_engine *e, int pi)
{
	struct pool *p = &e->peer_pools[pi];
	uint64_t bytes = e->cfg.host_arena_bytes;
	if (p->capacity && p->bytes + bytes > p->capacity)
		return NVS_E_HOST_OOM;
	/* That GPU's HBM is not ours alone: other clients back their slabs there too, and it may have
	 * clients of its own.  Claim the arena in the cross-process ledger first; no room to lend means
	 * the chunk goes to the next peer or to the host tier, like a peer that is simply full. */
	if (nvs_gl_lend(p->gl_dev, bytes, e->gl_reserve) != 0) {
		if (p->gl_refusals++ == 0)
			nvs_debug("engine: GPU %d has no HBM left to lend (ledger): spilling", p->device);
		return NVS_E_HOST_OOM;
	}
	struct arena *a = arena_new(bytes);
	if (!a) {
		nvs_gl_return(p->gl_dev, bytes);
		return NVS_E_HOST_OOM;
	}
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof(prop));
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = p->device;
	CUmemAccessDesc acc[2];
	memset(acc, 0, sizeof(acc));
	acc[0].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	acc[0].location.id = e->device;
	acc[0].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	acc[1].location = prop.location;
	acc[1].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	CUdeviceptr va = 0;
	if (e->d.MemCreate(&a->handle, bytes, &prop, 0) != CUDA_SUCCESS)
		goto fail;
	if (e->d.MemAddressReserve(&va, bytes, 0, 0, 0) != CUDA_SUCCESS) {
		e->d.MemRelease(a->handle);
		goto fail;
	}
	if (e->d.MemMap(va, bytes, 0, a->handle, 0) != CUDA_SUCCESS ||
	    e->d.MemSetAccess(va, bytes, acc, 2) != CUDA_SUCCESS) {
		e->d.MemUnmap(va, bytes);
		e->d.MemAddressFree(va, bytes);
		e->d.MemRelease(a->handle);
		goto fail;
	}
	a->dev_base = va;
	a->next = p->arenas;
	p->arenas = a;
	p->bytes += bytes;
	e->st.peer_pool_bytes += bytes;
	return 0;
fail:
	nvs_gl_return(p->gl_dev, bytes);
	arena_free(a);
	return NVS_E_HOST_OOM;
}

static uint64_t shp_reap_dead(struct shpool *sp);

/* Find backing for a chunk: peers first (striped), then pinned host.  e->mu held. */
static int backing_assign(nvs_engine *e, struct chunk *c, int nowait)
{
	if (c->backing)
		return 0;
	const uint32_t n = (uint32_t)(c->bytes / SLAB);
	const uint32_t tag = ++e->tag_next ? e->tag_next : ++e->tag_next; /* never 0 */
	memset(c->bvalid, 0, sizeof(c->bvalid));
	for (int t = 0; t < e->cfg.n_peers; ++t) {
		int pi = (int)((e->peer_rr + (uint32_t)t) % (uint32_t)e->cfg.n_peers);
		struct pool *p = &e->peer_pools[pi];
		if (pool_take(e, p, n, &c->backing, 0, tag) == 0 ||
		    (peer_pool_grow(e, pi) == 0 && pool_take(e, p, n, &c->backing, 0, tag) == 0)) {
			c->tier = (uint8_t)(TIER_PEER0 + pi);
			c->btag = tag;
			e->peer_rr = (uint32_t)pi + 1;
			e->st.peer_pool_used += c->bytes;
			return 0;
		}
	}
	double t0 = now_ms(), next_reap = 0;
	int overflow_failed = 0;
	for (;;) {
		if (pool_take(e, &e->host_pool, n, &c->backing, 0, tag) == 0)
			break;
		/* A private pool takes over retained copies before it pins more host memory; the shared
		 * pool first grows to its capacity (a budget fixed when it was created), then does. */
		if (!e->shp && e->cfg.retain &&
		    (pool_take(e, &e->host_pool, n, &c->backing, RS_PLAIN, tag) == 0 ||
		     pool_take(e, &e->host_pool, n, &c->backing, RS_STABLE, tag) == 0))
			break;
		/* pool empty: wait for the background pinning, or pin inline */
		int rc = host_pool_grow(e);
		if (rc == 0)
			continue;
		if (e->shp && e->cfg.retain &&
		    (pool_take(e, &e->host_pool, n, &c->backing, RS_PLAIN, tag) == 0 ||
		     pool_take(e, &e->host_pool, n, &c->backing, RS_STABLE, tag) == 0))
			break;
		if (!e->shp || nowait || now_ms() - t0 > e->cfg.oom_wait_ms)
			return rc;
		/* the shared pool is full and entirely pinned here: another client is about
		 * to hand units back (its fetch releases them batch by batch) -- unless it died.
		 * Whoever follows our release progress must not wait for us while we wait for it. */
		if (e->shp->hdr->releaser_pid == (int32_t)getpid())
			__atomic_store_n(&e->shp->hdr->releaser_pid, 0, __ATOMIC_RELEASE);
		if (now_ms() >= next_reap) {
			next_reap = now_ms() + 500;
			if (shp_reap_dead(e->shp))
				continue;
		}
		if (now_ms() - t0 >= e->pool_grace_ms && !overflow_failed) {
			if (host_pool_overflow(e) == 0)
				continue;
			overflow_failed = 1; /* no host memory either: keep waiting for units */
		}
		pthread_mutex_unlock(&e->mu);
		usleep(1000);
		pthread_mutex_lock(&e->mu);
	}
	c->tier = TIER_HOST;
	c->btag = tag;
	e->st.host_pool_used = e->host_pool.used;
	if (e->shp && e->cfg.prepin) {
		/* keep a few windows pinned ahead of the eviction front (pinning a window of
		 * the shared pool is ~10x faster than the eviction that fills it is not) */
		uint64_t want = e->host_pool.used + 8 * e->cfg.host_arena_bytes;
		if (want > e->pin_target) {
			e->pin_target = want;
			pthread_cond_signal(&e->pin_cv);
		}
	}
	return 0;
}

static struct pool *pool_of_tier(nvs_engine *e, uint8_t tier)
{
	return tier == TIER_HOST ? &e->host_pool : tier >= TIER_PEER0 ? &e->peer_pools[tier - TIER_PEER0] : NULL;
}

/* A RESIDENT chunk is about to rely on the backing copy it kept: is it still there?
 * 1: yes, and from now on nobody can take it (it is live again).  0: gone. */
static int backing_reclaim(nvs_engine *e, struct chunk *c)
{
	if (!c->retained)
		return c->backing != 0;
	c->retained = 0;
	e->st.retained_bytes -= c->bytes;
	struct pool *p = pool_of_tier(e, c->tier);
	if (p && c->backing && pool_reclaim(e, p, c->backing, (uint32_t)(c->bytes / SLAB), c->btag))
		return 1;
	/* somebody needed the units more: the copy is gone, the next eviction moves everything */
	c->backing = 0;
	c->tier = TIER_NONE;
	memset(c->bvalid, 0, sizeof(c->bvalid));
	e->st.host_pool_used = e->host_pool.used;
	return 0;
}

static void backing_release(nvs_engine *e, struct chunk *c)
{
	if (c->retained && !backing_reclaim(e, c))
		return;
	if (!c->backing)
		return;
	const uint32_t n = (uint32_t)(c->bytes / SLAB);
	if (c->tier == TIER_HOST) {
		pool_give(e, &e->host_pool, c->backing, n, c->btag);
		e->st.host_pool_used = e->host_pool.used;
	} else if (c->tier >= TIER_PEER0) {
		struct pool *p = &e->peer_pools[c->tier - TIER_PEER0];
		pool_give(e, p, c->backing, n, c->btag);
		e->st.peer_pool_used -= c->bytes;
		/* peer HBM is per-process (no shared pool yet): hand empty arenas back to the peer
		 * GPU at once, so that the client evicting right now finds room there */
		for (struct arena **pp = &p->arenas; *pp;) {
			struct arena *a = *pp;
			if (a->used != 0) {
				pp = &a->next;
				continue;
			}
			*pp = a->next;
			e->d.MemUnmap(a->dev_base, a->bytes);
			e->d.MemAddressFree(a->dev_base, a->bytes);
			e->d.MemRelease(a->handle);
			nvs_gl_return(p->gl_dev, a->bytes);
			p->bytes -= a->bytes;
			e->st.peer_pool_bytes -= a->bytes;
			arena_free(a);
		}
	}
	c->backing = 0;
	c->tier = TIER_NONE;
	memset(c->bvalid, 0, sizeof(c->bvalid));
}

/* The chunk is resident and its backing copy stays in the pool, reclaimable by anybody. */
static void backing_mark_retained(nvs_engine *e, struct chunk *c)
{
	if (!c->backing || c->retained || c->tier != TIER_HOST)
		return;
	pool_mark_retained(e, &e->host_pool, c->backing, (uint32_t)(c->bytes / SLAB),
			   c->stable == ST_STABLE ? RS_STABLE : RS_PLAIN);
	c->retained = 1;
	e->st.retained_bytes += c->bytes;
}

/*
 * A fetched chunk's backing copy: keep it or give it back?  Keeping costs host memory
 * that anybody may take over when the pool runs short, and buys an eviction that only
 * copies what changed.  Chunks that turned out dirty last time are not worth it --
 * except every VOLATILE_REPROBE-th time, to notice that they calmed down.
 */
static void backing_after_fetch(nvs_engine *e, struct chunk *c)
{
	if (!c->backing)
		return;
	int keep = e->cfg.retain && c->tier == TIER_HOST;
	if (keep && c->stable == ST_VOLATILE) {
		if (++c->volatile_skips < VOLATILE_REPROBE)
			keep = 0;
		else
			c->volatile_skips = 0;
	}
	if (!keep) {
		backing_release(e, c);
		return;
	}
	backing_mark_retained(e, c);
}

/* ------------------------------------------------------ shared pool ---- */

static void shp_close(nvs_engine *e)
{
	struct shpool *sp = e->shp;
	if (!sp)
		return;
	for (struct arena *a = e->host_pool.arenas, *nx; a; a = nx) {
		nx = a->next;
		if (a->shared) {
			e->d.MemHostUnregister(a->host_base);
		} else { /* overflow arena (host_pool_overflow) */
			e->d.MemFreeHost(a->host_base);
		}
		arena_free(a);
	}
	e->host_pool.arenas = NULL;
	if (sp->hdr)
		munmap(sp->hdr, SHP_HDR_BYTES + sp->hdr->capacity_slabs * SLAB);
	if (sp->fd >= 0)
		close(sp->fd);
	free(sp->registered);
	free(sp);
	e->shp = NULL;
}

/* Take back the units of clients that died without returning them (a killed
 * process cannot; one that exits normally does not bother).  Returns how many. */
static uint64_t shp_reap_dead(struct shpool *sp)
{
	uint64_t reaped = 0;
	int32_t last_pid = 0;
	int last_dead = 0;
	shp_lock(sp);
	for (uint64_t k = 0; k < sp->hdr->capacity_slabs; ++k) {
		int32_t pid = sp->hdr->owners[k];
		if (pid <= 0)
			continue;
		if (pid != last_pid) {
			last_pid = pid;
			last_dead = kill(pid, 0) != 0 && errno == ESRCH;
		}
		if (!last_dead)
			continue;
		sp->hdr->bitmap[k >> 6] &= ~(1ull << (k & 63));
		sp->hdr->owners[k] = 0;
		sp->hdr->rstate[k] = RS_NONE;
		sp->hdr->ctag[k] = 0;
		sp->hdr->used_slabs--;
		reaped++;
	}
	shp_unlock(sp);
	return reaped;
}

static uint64_t read_u64_file(const char *path, uint64_t dflt)
{
	FILE *f = fopen(path, "r");
	if (!f)
		return dflt;
	char buf[64] = "";
	uint64_t v = dflt;
	if (fgets(buf, sizeof(buf), f) && buf[0] >= '0' && buf[0] <= '9')
		v = strtoull(buf, NULL, 10);
	fclose(f);
	return v;
}

/* Host memory this process may still take: the memory cgroup's limit minus its usage (v2, then
 * v1), capped by MemAvailable.  UINT64_MAX when nothing can be read. */
static uint64_t host_memory_room(void)
{
	uint64_t room = UINT64_MAX;
	uint64_t lim = read_u64_file("/sys/fs/cgroup/memory.max", UINT64_MAX);
	uint64_t cur = read_u64_file("/sys/fs/cgroup/memory.current", 0);
	if (lim == UINT64_MAX) {
		lim = read_u64_file("/sys/fs/cgroup/memory/memory.limit_in_bytes", UINT64_MAX);
		cur = read_u64_file("/sys/fs/cgroup/memory/memory.usage_in_bytes", 0);
	}
	if (lim != UINT64_MAX && lim < (1ull << 60))
		room = lim > cur ? lim - cur : 0;
	FILE *f = fopen("/proc/meminfo", "r");
	if (f) {
		char line[128];
		while (fgets(line, sizeof(line), f)) {
			unsigned long long kb;
			if (sscanf(line, "MemAvailable: %llu kB", &kb) == 1) {
				if (kb * 1024ull < room)
					room = kb * 1024ull;
				break;
			}
		}
		fclose(f);
	}
	return room;
}

static uint64_t my_pid_ns(void)
{
	struct stat st;
	return stat("/proc/self/ns/pid", &st) == 0 ? (uint64_t)st.st_ino : 0;
}

/* Open (or create) the pool file.  Returns 0, or -1 to fall back to a private pool. */
static int shp_open(nvs_engine *e, const char *path, uint64_t capacity_bytes)
{
	struct shpool *sp = calloc(1, sizeof(*sp));
	if (!sp)
		return -1;
	snprintf(sp->path, sizeof(sp->path), "%s", path);
	const uint32_t window_slabs = (uint32_t)(e->cfg.host_arena_bytes / SLAB);
	uint64_t cap_slabs = capacity_bytes / SLAB / window_slabs * window_slabs;
	if (cap_slabs > SHP_MAX_SLABS)
		cap_slabs = SHP_MAX_SLABS / window_slabs * window_slabs;
	int creator = 1;
	if (access(path, F_OK) != 0) {
		/* Whoever creates the pool fixes its capacity, and with kept copies the pool WILL fill up
		 * to it.  A tmpfs smaller than the pool (docker's default /dev/shm is 64 MiB) would turn
		 * page faults into SIGBUS, a memory cgroup smaller than it (pinned and tmpfs pages are
		 * charged to it) into an OOM kill: shrink the
		 * budget to what the box can really give, and only fall back to private pools when that
		 * is less than a quarter of what was asked for. */
		char dir[256];
		snprintf(dir, sizeof(dir), "%s", path);
		char *slash = strrchr(dir, '/');
		if (slash)
			*slash = '\0';
		uint64_t room = host_memory_room();
		struct statvfs vfs;
		if (statvfs(slash ? dir : ".", &vfs) == 0 && (uint64_t)vfs.f_bavail * vfs.f_frsize < room)
			room = (uint64_t)vfs.f_bavail * vfs.f_frsize;
		const uint64_t reserve = e->cfg.shared_pool_bytes ? SHP_HDR_BYTES : (20ull << 30) + SHP_HDR_BYTES;
		const uint64_t fit = room > reserve ? (room - reserve) / SLAB / window_slabs * window_slabs : 0;
		if (fit < cap_slabs) {
			if (fit < cap_slabs / 4) {
				errno = ENOSPC;
				free(sp);
				return -1;
			}
			nvs_debug("engine: shared pool capacity cut from %" PRIu64 " to %" PRIu64 " GiB (host memory / tmpfs budget)",
				  (uint64_t)((cap_slabs * SLAB) >> 30), (uint64_t)((fit * SLAB) >> 30));
			cap_slabs = fit;
		}
	}
	sp->fd = open(path, O_RDWR | O_CREAT | O_EXCL | O_CLOEXEC | O_NOFOLLOW, 0600);
	if (sp->fd < 0 && errno == EEXIST) {
		creator = 0;
		sp->fd = open(path, O_RDWR | O_CLOEXEC | O_NOFOLLOW);
	}
	if (sp->fd < 0)
		goto fail;
	{
		/* The name is predictable and evicted GPU memory ends up in this file: only ever attach
		 * to a regular file that this very user created with mode 0600 (anybody able to plant
		 * such a file can already read our memory).  Otherwise: private pool. */
		struct stat st;
		if (creator)
			(void)fchmod(sp->fd, 0600); /* whatever the umask said */
		if (fstat(sp->fd, &st) != 0 || !S_ISREG(st.st_mode) || st.st_uid != geteuid() ||
		    (st.st_mode & 07777) != 0600 || st.st_nlink != 1) {
			nvs_warn("engine: %s is not a pool file of ours (owner %d, mode %o): not using it", path,
				 (int)st.st_uid, (unsigned)(st.st_mode & 07777));
			close(sp->fd);
			sp->fd = -1;
			creator = 0; /* it is somebody else's: do not unlink it either */
			errno = EPERM;
			goto fail;
		}
	}
	if (creator && ftruncate(sp->fd, (off_t)(SHP_HDR_BYTES + cap_slabs * SLAB)) != 0)
		goto fail;
	if (!creator) {
		/* wait for the creator to size and initialise the file */
		struct stat st;
		for (int i = 0; i < 5000; ++i) {
			if (fstat(sp->fd, &st) == 0 && (uint64_t)st.st_size > SHP_HDR_BYTES)
				break;
			usleep(1000);
		}
		if (fstat(sp->fd, &st) != 0 || (uint64_t)st.st_size <= SHP_HDR_BYTES)
			goto fail;
		cap_slabs = ((uint64_t)st.st_size - SHP_HDR_BYTES) / SLAB;
	}
	void *m = mmap(NULL, SHP_HDR_BYTES + cap_slabs * SLAB, PROT_READ | PROT_WRITE, MAP_SHARED, sp->fd, 0);
	if (m == MAP_FAILED)
		goto fail;
	sp->hdr = m;
	sp->data = (uint8_t *)m + SHP_HDR_BYTES;
	if (creator) {
		pthread_mutexattr_t at;
		pthread_mutexattr_init(&at);
		pthread_mutexattr_setpshared(&at, PTHREAD_PROCESS_SHARED);
		pthread_mutexattr_setrobust(&at, PTHREAD_MUTEX_ROBUST);
		pthread_mutex_init(&sp->hdr->mu, &at);
		pthread_mutexattr_destroy(&at);
		sp->hdr->version = SHP_VERSION;
		sp->hdr->window_slabs = window_slabs;
		sp->hdr->capacity_slabs = cap_slabs;
		sp->hdr->pid_ns = my_pid_ns();
		__atomic_store_n(&sp->hdr->magic, SHP_MAGIC, __ATOMIC_RELEASE);
	} else {
		for (int i = 0; i < 5000 && __atomic_load_n(&sp->hdr->magic, __ATOMIC_ACQUIRE) != SHP_MAGIC; ++i)
			usleep(1000);
		/* every field that later indexes the bitmap / owners arrays is checked against the file */
		if (sp->hdr->magic != SHP_MAGIC || sp->hdr->version != SHP_VERSION || sp->hdr->capacity_slabs != cap_slabs ||
		    cap_slabs > SHP_MAX_SLABS || sp->hdr->window_slabs == 0 || cap_slabs % sp->hdr->window_slabs != 0 ||
		    sp->hdr->used_slabs > cap_slabs || (uint64_t)sp->hdr->window_slabs * SLAB < e->cfg.chunk_bytes) {
			nvs_warn("engine: shared pool %s is not usable by this client (geometry/version)", path);
			munmap(m, SHP_HDR_BYTES + cap_slabs * SLAB);
			sp->hdr = NULL;
			goto fail;
		}
		if (sp->hdr->pid_ns != my_pid_ns()) {
			nvs_warn("engine: shared pool %s belongs to another pid namespace (its owners' liveness cannot be "
				 "checked from here): using a private pool", path);
			munmap(m, SHP_HDR_BYTES + cap_slabs * SLAB);
			sp->hdr = NULL;
			goto fail;
		}
		shp_reap_dead(sp);
	}
	sp->n_windows = (uint32_t)(cap_slabs / sp->hdr->window_slabs);
	sp->registered = calloc(sp->n_windows ? sp->n_windows : 1, 1);
	if (!sp->registered)
		goto fail;
	e->cfg.host_arena_bytes = (uint64_t)sp->hdr->window_slabs * SLAB;
	e->shp = sp;
	nvs_debug("engine: shared host pool %s: %" PRIu64 " GiB in %u windows (%s)", path, (uint64_t)((cap_slabs * SLAB) >> 30),
		  sp->n_windows, creator ? "created" : "attached");
	return 0;
fail:
	if (sp->hdr)
		munmap(sp->hdr, SHP_HDR_BYTES + cap_slabs * SLAB);
	if (sp->fd >= 0)
		close(sp->fd);
	if (creator && sp->fd >= 0)
		unlink(path);
	free(sp->registered);
	free(sp);
	return -1;
}

static void *pin_thread_main(void *arg)
{
	nvs_engine *e = arg;
	if (ctx_enter(e) != 0)
		return NULL;
	pthread_mutex_lock(&e->mu);
	while (!e->stopping) {
		if (e->host_pool.bytes >= e->pin_target) {
			pthread_cond_wait(&e->pin_cv, &e->mu);
			continue;
		}
		int rc = host_pool_grow(e);
		if (rc != 0) /* out of pinnable memory: stop trying, evict will report it */
			e->pin_target = e->host_pool.bytes;
	}
	pthread_mutex_unlock(&e->mu);
	ctx_leave(e);
	return NULL;
}

/* ----------------------------------------------------------- table ------ */

static unsigned hash_va(uint64_t va)
{
	return (unsigned)((va >> NVS_SLAB_SHIFT) * 0x9E3779B97F4A7C15ull >> (64 - HASH_BITS));
}

static struct alloc *table_find(nvs_engine *e, uint64_t va)
{
	for (struct alloc *a = e->buckets[hash_va(va)]; a; a = a->hnext)
		if (a->va == va)
			return a;
	return NULL;
}

/* index of the first allocation whose address is > va */
static size_t by_va_upper(const nvs_engine *e, uint64_t va)
{
	size_t lo = 0, hi = e->n_by_va;
	while (lo < hi) {
		size_t mid = (lo + hi) / 2;
		if (e->by_va[mid]->va <= va)
			lo = mid + 1;
		else
			hi = mid;
	}
	return lo;
}

static void table_insert(nvs_engine *e, struct alloc *a)
{
	if (e->n_by_va == e->cap_by_va) {
		size_t cap = e->cap_by_va ? 2 * e->cap_by_va : 256;
		struct alloc **nv = realloc(e->by_va, cap * sizeof(*nv));
		if (nv) {
			e->by_va = nv;
			e->cap_by_va = cap;
		}
	}
	if (e->n_by_va < e->cap_by_va) {
		size_t at = by_va_upper(e, a->va);
		memmove(&e->by_va[at + 1], &e->by_va[at], (e->n_by_va - at) * sizeof(*e->by_va));
		e->by_va[at] = a;
		e->n_by_va++;
	}
	unsigned h = hash_va(a->va);
	a->hnext = e->buckets[h];
	e->buckets[h] = a;
	a->prev = e->tail;
	a->next = NULL;
	if (e->tail)
		e->tail->next = a;
	else
		e->head = a;
	e->tail = a;
	e->st.n_allocs++;
	e->st.requested_bytes += a->req_bytes;
}

static void table_remove(nvs_engine *e, struct alloc *a)
{
	size_t at = by_va_upper(e, a->va);
	if (at > 0 && e->by_va[at - 1] == a) {
		memmove(&e->by_va[at - 1], &e->by_va[at], (e->n_by_va - at) * sizeof(*e->by_va));
		e->n_by_va--;
	}
	struct alloc **pp = &e->buckets[hash_va(a->va)];
	while (*pp && *pp != a)
		pp = &(*pp)->hnext;
	if (*pp)
		*pp = a->hnext;
	if (a->prev)
		a->prev->next = a->next;
	else
		e->head = a->next;
	if (a->next)
		a->next->prev = a->prev;
	else
		e->tail = a->prev;
	e->st.n_allocs--;
	e->st.requested_bytes -= a->req_bytes;
}

/* ------------------------------------------------------- map / unmap ---- */

static void state_account(nvs_engine *e, struct chunk *c, int new_state)
{
	uint64_t *from = c->state == CH_RESIDENT ? &e->st.resident_bytes
			 : c->state == CH_SWAPPED ? &e->st.swapped_bytes
						  : &e->st.unbacked_bytes;
	uint64_t *to = new_state == CH_RESIDENT ? &e->st.resident_bytes
		       : new_state == CH_SWAPPED ? &e->st.swapped_bytes
						 : &e->st.unbacked_bytes;
	*from -= c->bytes;
	*to += c->bytes;
	c->state = (uint8_t)new_state;
}

#define NVS_I_LOCK_LOST (-100) /* internal: chunk_map gave up because its owner no longer holds the GPU lock */

/* Give a chunk physical HBM.  Retries while another process is still releasing.
 * while_holding_lock: the caller is an allocation made by the lock HOLDER (mapped at once);
 * if the lock goes away while it waits for HBM, waiting on makes no sense -- nobody will be
 * asked to make room for a client that is not running -- so it returns NVS_I_LOCK_LOST and
 * the rest of the allocation stays virtual until the next fetch. */
static int chunk_map_ex(nvs_engine *e, struct chunk *c, double *wait_ms, int while_holding_lock);
static int chunk_map(nvs_engine *e, struct chunk *c, double *wait_ms)
{
	return chunk_map_ex(e, c, wait_ms, 0);
}

static int chunk_map_ex(nvs_engine *e, struct chunk *c, double *wait_ms, int while_holding_lock)
{
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof(prop));
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = e->device;
	CUmemAccessDesc acc;
	memset(&acc, 0, sizeof(acc));
	acc.location = prop.location;
	acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;

	double t0 = now_ms(), warned = 0, next_pressure = 0, last_progress = t0;
	size_t last_free = 0;
	for (;;) {
		CUresult r = e->d.MemCreate(&c->handle, c->bytes, &prop, 0);
		if (r == CUDA_SUCCESS)
			break;
		if (is_shutdown_error(r))
			return NVS_E_SHUTDOWN;
		if (r != CUDA_ERROR_OUT_OF_MEMORY) {
			nvs_warn("engine: cuMemCreate failed: %s", cu_name(e, r));
			return (int)r;
		}
		double waited = now_ms() - t0;
		if (waited > e->cfg.oom_wait_ms) {
			nvs_warn("engine: HBM still exhausted after %.0f ms", waited);
			return NVS_E_TIMEOUT;
		}
		if (!warned && waited > 2000) {
			nvs_debug("engine: waiting for HBM to be released by another client");
			warned = 1;
		}
		if (while_holding_lock && !e->resident_mode)
			return NVS_I_LOCK_LOST;
		if (e->cfg.pressure_cb && now_ms() - last_progress >= PRESSURE_AFTER_MS && waited >= next_pressure) {
			/* nobody is (any longer) freeing memory for us: say how much we still miss */
			e->cfg.pressure_cb(e->cfg.pressure_user, e->st.swapped_bytes + e->st.unbacked_bytes);
			next_pressure = waited + 1000;
		}
		/* Wait until the driver reports room for this chunk before trying again: a
		 * failing cuMemCreate is expensive and serialises with the cuMemRelease
		 * calls of the process that is evicting. */
		pthread_mutex_unlock(&e->mu); /* api_mu still serialises the entry points; let stats / pinning run */
		for (int spin = 0; spin < 20; ++spin) {
			size_t free_b = 0, total_b = 0;
			usleep(1000);
			if (e->d.MemGetInfo(&free_b, &total_b) != CUDA_SUCCESS)
				break;
			if (free_b > last_free)
				last_progress = now_ms(); /* somebody is handing HBM back right now */
			last_free = free_b;
			if (free_b >= c->bytes + (64u << 20))
				break;
		}
		pthread_mutex_lock(&e->mu);
	}
	if (wait_ms)
		*wait_ms += now_ms() - t0;
	CUresult r = e->d.MemMap(c->va, c->bytes, 0, c->handle, 0);
	if (r == CUDA_SUCCESS)
		r = e->d.MemSetAccess(c->va, c->bytes, &acc, 1);
	if (r != CUDA_SUCCESS) {
		nvs_warn("engine: cuMemMap/cuMemSetAccess failed: %s", cu_name(e, r));
		e->d.MemUnmap(c->va, c->bytes);
		e->d.MemRelease(c->handle);
		return (int)r;
	}
	return 0;
}

static int chunk_unmap(nvs_engine *e, struct chunk *c)
{
	CUresult r = e->d.MemUnmap(c->va, c->bytes);
	if (r == CUDA_SUCCESS)
		r = e->d.MemRelease(c->handle);
	c->handle = 0;
	if (is_shutdown_error(r))
		return NVS_E_SHUTDOWN;
	if (r != CUDA_SUCCESS)
		nvs_warn("engine: cuMemUnmap/cuMemRelease failed: %s", cu_name(e, r));
	return (int)r;
}

/* ------------------------------------------------------------ launch ---- */

static uint32_t grid_for(nvs_engine *e, uint32_t want, int peer_traffic)
{
	if (want)
		return want;
	if (e->cfg.copy_grid)
		return e->cfg.copy_grid;
	return peer_traffic ? (uint32_t)(e->n_sms / 2) : 8u;
}

/* Enqueue one copy of n descriptors (device-visible array) on e->stream. */
static int launch_descs(nvs_engine *e, uint64_t descs_dev, const nvs_copy_desc *descs_host, uint32_t n,
			uint32_t variant, uint32_t grid)
{
	int rc = 0;
	if (n == 0)
		return 0;
	if (variant == NVS_COPY_CE) {
		for (uint32_t i = 0; i < n; ++i)
			CK(e, e->d.MemcpyAsync(descs_host[i].dst, descs_host[i].src, descs_host[i].bytes, e->stream));
		return 0;
	}
	if (e->counter_next == N_COUNTERS) {
		CK(e, e->d.MemsetD32Async(e->counters, 0, N_COUNTERS, e->stream));
		e->counter_next = 0;
	}
	CUdeviceptr counter = e->counters + 4ull * e->counter_next++;
	uint32_t n_descs = n;
	if (variant == NVS_COPY_TMA) {
		uint32_t tile = e->cfg.tma_tile_bytes, stages = e->cfg.tma_stages, warps = e->cfg.tma_warps;
		void *params[] = {&descs_dev, &n_descs, &counter, &tile, &stages};
		CK(e, e->d.LaunchKernel(e->fn_tma, grid, 1, 1, 32 * warps, 1, 1, warps * stages * tile,
					e->stream, params, NULL));
	} else {
		void *params[] = {&descs_dev, &n_descs, &counter};
		CK(e, e->d.LaunchKernel(e->fn_ldg, grid, 1, 1, e->cfg.ldg_threads, 1, 1, 0, e->stream, params,
					NULL));
	}
	e->st.kernel_launches_total++;
out:
	return rc;
}

static void slot_reset(struct slot *s)
{
	s->n_descs = 0;
	s->n_ce = 0;
	s->n_chunks = 0;
	s->n_aux = 0;
	s->peer_traffic = 0;
}

static inline int slab_is_const(const struct chunk *c, uint32_t i)
{
	return (c->cmask[i >> 6] >> (i & 63)) & 1;
}

static inline int mask_get(const uint64_t *m, uint32_t i)
{
	return (m[i >> 6] >> (i & 63)) & 1;
}

static inline void mask_set(uint64_t *m, uint32_t i)
{
	m[i >> 6] |= 1ull << (i & 63);
}

static void mask_fill(uint64_t *m, uint32_t n)
{
	memset(m, 0, sizeof(uint64_t) * (MAX_CHUNK_SLABS / 64));
	for (uint32_t i = 0; i < n; ++i)
		mask_set(m, i);
}

/* Which engine moves a chunk between HBM and its backing tier?  Over PCIe a copy-engine transfer
 * carries 256-byte TLPs, an SM-issued one 128-byte TLPs, so the pinned-host tier moves on the copy
 * engines and the SMs do what those cannot (scan, hash, splat).  Over NVLink the kernel, which keeps
 * many more bytes in flight than per-chunk cuMemcpyAsync calls, moves both directions. */
/* one launch consumes the whole kernel list of a slot: the peer tier's kernel if it has one */
static uint32_t kernel_variant(const nvs_engine *e, int to_backing)
{
	const uint32_t peer = to_backing ? e->cfg.peer_evict_variant : e->cfg.peer_fetch_variant;
	const uint32_t host = to_backing ? e->cfg.evict_variant : e->cfg.fetch_variant;
	return peer != NVS_COPY_CE ? peer : host != NVS_COPY_CE ? host : NVS_COPY_TMA;
}

static uint32_t variant_for(const nvs_engine *e, uint8_t tier, int to_backing)
{
	if (tier >= TIER_PEER0)
		return to_backing ? e->cfg.peer_evict_variant : e->cfg.peer_fetch_variant;
	return to_backing ? e->cfg.evict_variant : e->cfg.fetch_variant;
}

/* Copy descriptors for the slabs of `c` selected by `mask`.  Kernel variants get one
 * descriptor per slab; the copy engines get one per run of adjacent slabs (a chunk's
 * backing is contiguous). */
static int slot_push_chunk(nvs_engine *e, struct slot *s, struct chunk *c, int to_backing, const uint64_t *mask)
{
	if (s->n_chunks == s->cap_chunks)
		return -1;
	s->chunks[s->n_chunks++] = c;
	const uint32_t variant = variant_for(e, c->tier, to_backing);
	const uint32_t n = (uint32_t)(c->bytes / SLAB);
	for (uint32_t i = 0; i < n;) {
		if (!mask_get(mask, i)) {
			++i;
			continue;
		}
		uint32_t run = 1;
		nvs_copy_desc *d;
		if (variant == NVS_COPY_CE) {
			while (i + run < n && mask_get(mask, i + run))
				++run;
			if (s->n_ce == s->cap_ce)
				return -1;
			d = &s->ce[s->n_ce++];
		} else {
			if (s->n_descs == s->cap_descs)
				return -1;
			d = &s->descs[s->n_descs++];
			s->peer_traffic |= c->tier >= TIER_PEER0;
		}
		const uint64_t off = (uint64_t)i * SLAB;
		d->src = (to_backing ? c->va : c->backing) + off;
		d->dst = (to_backing ? c->backing : c->va) + off;
		d->bytes = (uint64_t)run * SLAB;
		d->tag = (c->va + off) >> NVS_SLAB_SHIFT;
		i += run;
	}
	return 0;
}

/* Enqueue everything a slot has gathered on e->stream: one sm_90a kernel launch for the
 * kernel list, one cuMemcpyAsync per run of the copy-engine list. */
static int slot_launch(nvs_engine *e, struct slot *s, uint32_t kernel_variant, nvs_xfer_report *rep)
{
	int rc = 0;
	if (s->n_descs) {
		if ((rc = launch_descs(e, s->descs_dev, s->descs, s->n_descs, kernel_variant,
				       grid_for(e, 0, s->peer_traffic))) != 0)
			return rc;
		rep->launches++;
	}
	if (s->n_ce) {
		if ((rc = launch_descs(e, 0, s->ce, s->n_ce, NVS_COPY_CE, 0)) != 0)
			return rc;
		rep->ce_calls += s->n_ce;
		e->st.ce_calls_total += s->n_ce;
	}
	return 0;
}

static int launch_aux(nvs_engine *e, CUfunction fn, struct slot *s, CUstream stream, int with_out, uint32_t want_hash)
{
	int rc = 0;
	if (s->n_aux == 0)
		return 0;
	if (e->scan_counter_next == N_COUNTERS) {
		CK(e, e->d.MemsetD32Async(e->counters + 4ull * N_COUNTERS, 0, N_COUNTERS, stream));
		e->scan_counter_next = 0;
	}
	CUdeviceptr counter = e->counters + 4ull * (N_COUNTERS + e->scan_counter_next++);
	uint32_t n = s->n_aux;
	/* 256 threads per CTA is part of the hash's definition (lane = thread) */
	unsigned per_sm = with_out ? 4u : 8u;
	unsigned grid = n < (unsigned)e->n_sms * per_sm ? n : (unsigned)e->n_sms * per_sm;
	void *p_scan[] = {&s->aux_dev, &n, &counter, &s->scan_out_dev, &want_hash};
	void *p_splat[] = {&s->aux_dev, &n, &counter};
	CK(e, e->d.LaunchKernel(fn, grid, 1, 1, 256, 1, 1, 0, stream, with_out ? p_scan : p_splat, NULL));
	e->st.kernel_launches_total++;
out:
	return rc;
}

/*
 * Look at the chunks gathered in `s` before they leave HBM: one pass of the scan kernel
 * tells, per slab, whether it is same-filled (described by 8 bytes, not moved) and -- with
 * retention on -- its 128-bit content hash, from which follows what this eviction has to
 * copy (c->cpmask): every slab that is neither same-filled nor identical to what the
 * chunk's retained backing copy already holds.
 */
static int scan_slot(nvs_engine *e, struct slot *s, nvs_xfer_report *rep)
{
	int rc = 0;
	const uint32_t want_hash = e->cfg.retain ? 1u : 0u;
	s->n_aux = 0;
	uint64_t bytes = 0;
	for (uint32_t k = 0; k < s->n_chunks; ++k) {
		struct chunk *c = s->chunks[k];
		for (uint64_t off = 0; off < c->bytes; off += SLAB) {
			if (s->n_aux == s->cap_aux)
				return NVS_E_BAD_ARG;
			nvs_copy_desc *d = &s->aux[s->n_aux++];
			d->src = c->va + off;
			d->dst = 0;
			d->bytes = SLAB;
			d->tag = 0;
		}
		bytes += c->bytes;
	}
	CK(e, e->d.EventRecord(e->scan_begin, e->scan_stream));
	if ((rc = launch_aux(e, e->fn_scan, s, e->scan_stream, 1, want_hash)) != 0)
		return rc;
	CK(e, e->d.EventRecord(e->scan_done, e->scan_stream));
	CK(e, e->d.EventSynchronize(e->scan_done));
	{
		float ms = 0;
		if (e->d.EventElapsedTime(&ms, e->scan_begin, e->scan_done) == CUDA_SUCCESS)
			rep->scan_ms += ms;
		rep->launches++;
		rep->scan_launches++;
		/* the early-exit scan reads one 32 KiB tile of a slab that is not same-filled */
		rep->scanned_bytes += want_hash ? bytes : 0;
	}
	uint32_t at = 0;
	for (uint32_t k = 0; k < s->n_chunks; ++k) {
		struct chunk *c = s->chunks[k];
		const uint32_t n = (uint32_t)(c->bytes / SLAB);
		memset(c->cmask, 0, sizeof(c->cmask));
		memset(c->cpmask, 0, sizeof(c->cpmask));
		c->n_const = 0;
		c->est_copy = 0;
		if (want_hash && !c->nh && !(c->nh = malloc(MAX_CHUNK_SLABS * sizeof(struct slab_hash))))
			return NVS_E_HOST_OOM;
		for (uint32_t i = 0; i < n; ++i, ++at) {
			const struct scan_result *r = &s->scan_out[at];
			if (want_hash) {
				c->nh[i].h0 = r->h0;
				c->nh[i].h1 = r->h1;
			}
			if (r->is_const && e->cfg.elide_constant) {
				if (!c->cvals && !(c->cvals = calloc(MAX_CHUNK_SLABS, sizeof(uint64_t))))
					return NVS_E_HOST_OOM;
				c->cvals[i] = r->value;
				mask_set(c->cmask, i);
				c->n_const++;
				if (!want_hash)
					rep->scanned_bytes += SLAB;
				continue;
			}
			if (!want_hash)
				rep->scanned_bytes += 32768;
			if (want_hash && c->had_backing && c->hash && mask_get(c->bvalid, i) &&
			    c->hash[i].h0 == r->h0 && c->hash[i].h1 == r->h1)
				continue; /* the backing copy of this slab is still good */
			mask_set(c->cpmask, i);
			c->est_copy += SLAB;
		}
		c->scanned = 1;
	}
out:
	return rc;
}

/* ------------------------------------------------------------- evict ---- */

/*
 * Victim order of a partial eviction.  Every chunk has to be resident again before its
 * owner may run (VMM memory cannot fault), so WHICH chunks are out never costs a miss
 * later: what differs between chunks is what it costs to put them out now.  Cheapest
 * first -- chunks whose retained backing copy is still valid or that are same-filled go
 * for free -- then the ones the host side has not written for longest (nvs_touch), then
 * least recently fetched; the address only breaks ties.
 */
static int cmp_chunk_victim(const void *a, const void *b)
{
	const struct chunk *x = *(struct chunk *const *)a, *y = *(struct chunk *const *)b;
	if (x->est_copy != y->est_copy)
		return x->est_copy < y->est_copy ? -1 : 1;
	if (x->touch != y->touch)
		return x->touch < y->touch ? -1 : 1;
	if (x->epoch != y->epoch)
		return x->epoch < y->epoch ? -1 : 1;
	return x->va < y->va ? -1 : x->va > y->va;
}

static void report_emit(nvs_engine *e, const char *what, const nvs_xfer_report *r, int favour)
{
	nvs_debug("engine: %s %" PRIu64 " MiB (+%" PRIu64 " MiB same-filled, +%" PRIu64 " MiB clean: not moved) in %.1f ms "
		  "(copy %.1f ms = %.1f GB/s, map %.1f ms, wait %.1f ms, scan %.1f ms)", what, r->bytes >> 20,
		  r->elided_bytes >> 20, r->clean_bytes >> 20, r->wall_ms, r->copy_ms,
		  r->copy_ms > 0 ? r->bytes / 1e6 / r->copy_ms : 0.0, r->map_ms, r->wait_ms, r->scan_ms);
	if (!e->stats_file)
		return;
	/* peer tier: what the cross-process ledger says about the GPUs we back our slabs on, next to what we
	 * hold there ourselves (all clients' arenas together must be what those GPUs have "lent") */
	char gl[160] = "";
	if (e->cfg.n_peers > 0) {
		uint64_t lent = 0, mine = 0, refused = 0;
		int tracked = 0;
		for (int i = 0; i < e->cfg.n_peers; ++i) {
			const struct pool *p = &e->peer_pools[i];
			tracked += p->gl_dev >= 0;
			lent += nvs_gl_lent(p->gl_dev);
			mine += nvs_gl_mine(p->gl_dev, NVS_GL_LENT);
			refused += p->gl_refusals;
		}
		snprintf(gl, sizeof(gl), ",\"peer_pool_bytes\":%" PRIu64 ",\"gl_tracked_peers\":%d,\"gl_lent\":%" PRIu64
			 ",\"gl_my_lent\":%" PRIu64 ",\"gl_refusals\":%" PRIu64, e->st.peer_pool_bytes, tracked, lent, mine, refused);
	}
	fprintf(e->stats_file,
		"{\"op\":\"%s\",\"t\":%.6f,\"pid\":%d,\"bytes\":%" PRIu64 ",\"slabs\":%" PRIu64
		",\"chunks\":%" PRIu64 ",\"launches\":%" PRIu64 ",\"ce_calls\":%" PRIu64 ",\"wall_ms\":%.3f,\"copy_ms\":%.3f,"
		"\"map_ms\":%.3f,\"wait_ms\":%.3f,\"scan_ms\":%.3f,\"host_bytes\":%" PRIu64 ",\"peer_bytes\":%" PRIu64
		",\"elided_bytes\":%" PRIu64 ",\"clean_bytes\":%" PRIu64 ",\"scanned_bytes\":%" PRIu64
		",\"scan_launches\":%" PRIu64 ",\"retained_bytes\":%" PRIu64 ",\"pool_used\":%" PRIu64 ",\"favour\":%d%s}\n",
		what, wall_s(), (int)getpid(), r->bytes, r->slabs, r->chunks, r->launches, r->ce_calls, r->wall_ms, r->copy_ms,
		r->map_ms, r->wait_ms, r->scan_ms, r->host_bytes, r->peer_bytes, r->elided_bytes, r->clean_bytes,
		r->scanned_bytes, r->scan_launches, e->st.retained_bytes, e->host_pool.used, favour, gl);
	fflush(e->stats_file);
}

/* forget what this eviction learned about a chunk (it stays resident, or the eviction failed) */
static void scan_forget(struct chunk *c)
{
	free(c->nh);
	c->nh = NULL;
	c->scanned = 0;
	c->had_backing = 0;
	c->est_copy = 0;
	if (c->state == CH_RESIDENT) {
		memset(c->cmask, 0, sizeof(c->cmask));
		c->n_const = 0;
	}
}

/* wait for a slot's copy, then give its chunks' HBM back */
static int evict_retire(nvs_engine *e, struct slot *s, nvs_xfer_report *rep)
{
	int rc = 0;
	if (!s->busy)
		return 0;
	CK(e, e->d.EventSynchronize(s->done));
	{
		float ms = 0;
		if ((s->n_descs || s->n_ce) && e->d.EventElapsedTime(&ms, s->begin, s->done) == CUDA_SUCCESS)
			rep->copy_ms += ms;
	}
	double t0 = now_ms();
	for (uint32_t i = 0; i < s->n_chunks; ++i) {
		struct chunk *c = s->chunks[i];
		const uint32_t n = (uint32_t)(c->bytes / SLAB);
		int r = chunk_unmap(e, c);
		if (r != 0 && rc == 0)
			rc = r;
		state_account(e, c, CH_SWAPPED);
		/* what the backing copy holds now, slab by slab: the bytes just copied, or the bytes that
		 * were already there and still match; same-filled slabs have no bytes there at all */
		if (c->nh && c->backing) {
			if (!c->hash)
				c->hash = malloc(MAX_CHUNK_SLABS * sizeof(struct slab_hash));
			if (c->hash) {
				for (uint32_t k = 0; k < n; ++k)
					if (mask_get(c->cpmask, k))
						c->hash[k] = c->nh[k];
				for (uint32_t k = 0; k < MAX_CHUNK_SLABS / 64; ++k)
					c->bvalid[k] = ~c->cmask[k];
			} else {
				memset(c->bvalid, 0, sizeof(c->bvalid));
			}
		} else {
			memset(c->bvalid, 0, sizeof(c->bvalid));
		}
		if (c->had_backing) /* worth keeping a copy of: at most half of it had changed */
			c->stable = 2 * c->est_copy <= c->bytes - (uint64_t)c->n_const * SLAB ? ST_STABLE : ST_VOLATILE;
		free(c->nh);
		c->nh = NULL;
		c->scanned = 0;
		c->had_backing = 0;
		rep->chunks++;
	}
	rep->map_ms += now_ms() - t0;
	if (e->shp && e->shp->hdr->releaser_pid == (int32_t)getpid()) {
		uint64_t freed = 0;
		for (uint32_t i = 0; i < s->n_chunks; ++i)
			freed += s->chunks[i]->bytes;
		__atomic_fetch_add(&e->shp->hdr->released_bytes, freed, __ATOMIC_RELEASE);
	}
out:
	s->busy = 0;
	slot_reset(s);
	return rc;
}

/* The owner is about to give the lock away and will then evict: said BEFORE the next holder is
 * told to go, so that its fetch knows somebody is releasing HBM for it and follows the progress
 * words in the shared pool header instead of polling the driver. */
void nvs_evict_announce(nvs_engine *e)
{
	if (!e || !e->shp)
		return;
	struct shp_hdr *h = e->shp->hdr;
	h->released_bytes = 0;
	__atomic_fetch_add(&h->release_seq, 1, __ATOMIC_RELEASE);
	__atomic_store_n(&h->releaser_pid, (int32_t)getpid(), __ATOMIC_RELEASE);
}

static void evict_announce_done(nvs_engine *e)
{
	if (e->shp && e->shp->hdr->releaser_pid == (int32_t)getpid())
		__atomic_store_n(&e->shp->hdr->releaser_pid, 0, __ATOMIC_RELEASE);
}

static int evict_impl(nvs_engine *e, uint64_t min_bytes, nvs_xfer_report *rep_out, int best_effort);

int nvs_evict(nvs_engine *e, uint64_t min_bytes, nvs_xfer_report *rep_out)
{
	return evict_impl(e, min_bytes, rep_out, 0);
}

int nvs_evict_best_effort(nvs_engine *e, uint64_t min_bytes, nvs_xfer_report *rep_out)
{
	return evict_impl(e, min_bytes, rep_out, 1);
}

/* scan `n` chunks (which all fit one slot; the slot is empty) unless this eviction has done so already */
static int scan_chunks(nvs_engine *e, struct slot *s, struct chunk **cs, uint32_t n, nvs_xfer_report *rep)
{
	uint32_t m = 0;
	int rc = 0;
	if (s->n_chunks != 0 || n > s->cap_chunks)
		return NVS_E_BAD_ARG;
	for (uint32_t k = 0; k < n; ++k) {
		struct chunk *c = cs[k];
		if (c->scanned)
			continue;
		/* does it still have the backing copy it kept?  (from here on nobody can take it) */
		c->had_backing = (uint8_t)(c->backing && backing_reclaim(e, c));
		s->chunks[m++] = c;
	}
	if (m) {
		s->n_chunks = m;
		rc = scan_slot(e, s, rep);
	}
	s->n_chunks = 0;
	return rc;
}

static int evict_impl(nvs_engine *e, uint64_t min_bytes, nvs_xfer_report *rep_out, int best_effort)
{
	nvs_xfer_report rep;
	memset(&rep, 0, sizeof(rep));
	if (!e)
		return NVS_E_BAD_ARG;
	int rc = 0;
	struct chunk **victims = NULL;
	double t_begin = now_ms();
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);

	size_t n_res = 0, n_all = 0, n_vict = 0;
	uint64_t resident = 0;
	for (struct alloc *a = e->head; a; a = a->next)
		if (!a->passthrough)
			n_res += a->n_chunks;
	victims = malloc((n_res ? n_res : 1) * sizeof(*victims));
	if (!victims) {
		rc = NVS_E_HOST_OOM;
		goto out;
	}
	for (struct alloc *a = e->head; a; a = a->next) {
		if (a->passthrough)
			continue;
		for (uint32_t i = 0; i < a->n_chunks; ++i)
			if (a->chunks[i].state == CH_RESIDENT) {
				victims[n_all++] = &a->chunks[i];
				resident += a->chunks[i].bytes;
				a->chunks[i].est_copy = 0;
			}
	}
	n_vict = n_all;
	const int can_scan = e->cfg.elide_constant || e->cfg.retain;
	if (min_bytes && min_bytes < resident) {
		/* a partial eviction chooses: learn first what each chunk would cost (one pass of the
		 * scan kernel over everything resident, at HBM speed), then take the cheapest */
		if (can_scan) {
			struct slot *s = &e->slots[0];
			for (size_t i = 0; i < n_all;) {
				uint32_t n = 0;
				uint64_t b = 0;
				while (i + n < n_all && n < s->cap_chunks && (b + victims[i + n]->bytes) / SLAB <= s->cap_aux &&
				       b < 4 * e->cfg.batch_bytes) {
					b += victims[i + n]->bytes;
					++n;
				}
				if ((rc = scan_chunks(e, s, &victims[i], n, &rep)) != 0)
					goto out;
				i += n;
			}
		}
		qsort(victims, n_all, sizeof(*victims), cmp_chunk_victim);
		uint64_t acc = 0;
		size_t k = 0;
		while (k < n_all && acc < min_bytes)
			acc += victims[k++]->bytes;
		n_vict = k;
		/* the rest stays: a backing copy it had validated goes back to being reclaimable */
		for (size_t j = n_vict; j < n_all; ++j) {
			struct chunk *c = victims[j];
			const int had = c->had_backing;
			scan_forget(c);
			if (had)
				backing_mark_retained(e, c);
		}
	}

	unsigned batch_no = 0;
	size_t i = 0;
	while (i < n_vict) {
		struct slot *s = &e->slots[batch_no % N_SLOTS];
		if ((rc = evict_retire(e, s, &rep)) != 0)
			goto out;
		uint64_t batch = 0, copied = 0;
		/* 1. which chunks, 2. what do their slabs need, 3. backing + descriptors */
		struct chunk **picked = &victims[i];
		uint32_t n_picked = 0;
		while (i < n_vict && batch < e->cfg.batch_bytes && n_picked < s->cap_chunks &&
		       (batch + victims[i]->bytes) / SLAB <= s->cap_descs) {
			batch += victims[i]->bytes;
			++n_picked;
			++i;
		}
		if (can_scan) {
			if ((rc = scan_chunks(e, s, picked, n_picked, &rep)) != 0)
				goto out;
		} else {
			for (uint32_t k = 0; k < n_picked; ++k) {
				struct chunk *c = picked[k];
				c->had_backing = (uint8_t)(c->backing && backing_reclaim(e, c));
				mask_fill(c->cpmask, (uint32_t)(c->bytes / SLAB));
				c->est_copy = c->bytes;
				c->scanned = 1;
			}
		}
		int tier_full = 0, must_drain = 0, any_busy = 0;
		for (unsigned q = 0; q < N_SLOTS; ++q)
			any_busy |= e->slots[q].busy;
		for (uint32_t k = 0; k < n_picked; ++k) {
			struct chunk *c = picked[k];
			const uint32_t n = (uint32_t)(c->bytes / SLAB);
			const uint64_t moving = c->est_copy;
			if (c->n_const == n && c->backing)
				backing_release(e, c); /* nothing but same-filled slabs: 8 bytes each describe it */
			/* Only wait for room in the backing tier with nothing of ours in flight: the units we
			 * wait for come back when another client fetches, and it can only fetch into the HBM
			 * that our already-copied batches still hold until they are retired. */
			const int nowait = best_effort || k > 0 || any_busy;
			if (c->n_const != n && !c->backing && (rc = backing_assign(e, c, nowait)) != 0) {
				if (!(nowait && rc == NVS_E_HOST_OOM))
					goto out;
				/* the tier is full: this chunk and the rest of the batch stay where they are ... */
				rc = 0;
				if (best_effort) {
					tier_full = 1; /* ... for good */
				} else {
					must_drain = 1; /* ... until what is in flight has left HBM; then we come back to them */
					i -= n_picked - k;
				}
				break;
			}
			if (slot_push_chunk(e, s, c, 1, c->cpmask) != 0) {
				rc = NVS_E_BAD_ARG;
				goto out;
			}
			copied += moving;
			if (c->tier >= TIER_PEER0)
				rep.peer_bytes += moving;
			else
				rep.host_bytes += moving;
			rep.elided_bytes += (uint64_t)c->n_const * SLAB;
			rep.clean_bytes += c->bytes - (uint64_t)c->n_const * SLAB - moving;
		}
		if (s->n_chunks) {
			CK(e, e->d.EventRecord(s->begin, e->stream));
			if ((rc = slot_launch(e, s, kernel_variant(e, 1), &rep)) != 0)
				goto out;
			CK(e, e->d.EventRecord(s->done, e->stream));
			s->busy = 1;
			rep.bytes += copied;
			rep.slabs += copied / SLAB;
			batch_no++;
		}
		if (tier_full)
			break;
		if (must_drain) /* release the HBM of every batch copied so far before waiting for units */
			for (unsigned q = 0; q < N_SLOTS; ++q)
				if ((rc = evict_retire(e, &e->slots[q], &rep)) != 0)
					goto out;
	}
	for (unsigned k = 0; k < N_SLOTS; ++k) {
		int r = evict_retire(e, &e->slots[(batch_no + k) % N_SLOTS], &rep);
		if (r != 0 && rc == 0)
			rc = r;
	}
	if (min_bytes == 0 && e->st.resident_bytes == 0)
		e->resident_mode = 0; /* everything is out: the owner no longer holds the GPU */
	e->st.n_evicts++;
	e->st.evicted_bytes_total += rep.bytes;
	e->st.clean_skipped_bytes_total += rep.clean_bytes;
out:
	if (rc != 0) /* never leave copies in flight behind an error */
		e->d.StreamSynchronize(e->stream);
	for (unsigned k = 0; k < N_SLOTS; ++k) {
		e->slots[k].busy = 0;
		slot_reset(&e->slots[k]);
	}
	evict_announce_done(e);
	/* chunks this call looked at but did not put out (it stopped early, or failed) */
	for (size_t j = 0; victims && j < n_all; ++j) {
		struct chunk *c = victims[j];
		if (c->state == CH_RESIDENT && (c->scanned || c->nh || c->had_backing)) {
			const int had = c->had_backing;
			scan_forget(c);
			if (had)
				backing_mark_retained(e, c);
		}
	}
	rep.wall_ms = now_ms() - t_begin;
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	free(victims);
	if (rc == 0 && (rep.bytes || rep.elided_bytes || rep.clean_bytes))
		report_emit(e, "evict", &rep, best_effort); /* favour: done on a pressure hint, not at a hand-off */
	if (rep_out)
		*rep_out = rep;
	return rc;
}

/* ------------------------------------------------------------- fetch ---- */

/*
 * Burst gating.  While another process is still handing its HBM back, do NOT map
 * each chunk the moment it fits: with HBM full, one process releasing and another
 * creating chunk by chunk slow every VMM call down by an order of magnitude, below the
 * PCIe copy it is supposed to feed; one process at a time runs at full speed.  Round 1
 * therefore mapped in fixed 8 GiB bursts.
 *
 * Round 2: since unchanged slabs are no longer copied, most of an eviction is a bare
 * release that takes ~0.1 s for 70 GB -- if nobody interferes.  So the gate now follows
 * the releaser instead of a byte count: wait while the free HBM is still GROWING, go as
 * soon as it has stood still for NVS_SETTLE_MS with room for a batch (the releaser is
 * done, or is busy copying the next dirty batch: a chunk every ~5 ms over PCIe, and then
 * its few VMM calls hardly collide with ours), or as soon as `burst_bytes` (now a cap:
 * 64 GiB) or everything still missing is free.  Measured on the BASELINE configuration
 * (r2 calls 1 -> 2): fetch wall 2.21 s with fixed 8 GiB bursts (copy 1.81 s + 0.40 s of
 * stalls), see DESIGN.md section 7 for the adaptive gate.
 */
#define NVS_SETTLE_MS 3.0
static int fetch_retire(nvs_engine *e, struct slot *s, nvs_xfer_report *rep);

/* While a fetch waits for HBM: hand back the backing units of batches that have already
 * landed.  The client that is evicting into a tight pool may be waiting for exactly those
 * units, and we may be waiting for the HBM its eviction frees. */
static void fetch_retire_completed(nvs_engine *e, nvs_xfer_report *rep)
{
	for (unsigned k = 0; k < N_SLOTS; ++k) {
		struct slot *s = &e->slots[k];
		if (s->busy && e->d.EventQuery(s->done) == CUDA_SUCCESS)
			fetch_retire(e, s, rep);
	}
}

static int wait_for_hbm_burst(nvs_engine *e, uint64_t remaining, nvs_xfer_report *rep)
{
	/* head-room kept below the releasing client's own margin (1/512 of the HBM, client.c) */
	const uint64_t slack = e->cfg.chunk_bytes < (64ull << 20) ? e->cfg.chunk_bytes : (64ull << 20);
	const uint64_t one_batch = e->cfg.batch_bytes + e->cfg.chunk_bytes + slack;
	const uint64_t cap = remaining < e->cfg.burst_bytes ? remaining : e->cfg.burst_bytes;
	size_t free_b = 0, total_b = 0;
	if (e->d.MemGetInfo(&free_b, &total_b) != CUDA_SUCCESS || free_b >= remaining + slack)
		return 0; /* everything that is still missing fits: nobody has to release anything for us */
	double t0 = now_ms(), next_pressure = 0, last_growth = t0;
	size_t last_free = free_b;
	int polls = 0;
	/* Somebody has announced that it is releasing for us (same scheduler, shared pool): follow
	 * its progress words, without a single driver call, until it is done or `cap` has come back. */
	if (e->shp) {
		struct shp_hdr *h = e->shp->hdr;
		int32_t who = __atomic_load_n(&h->releaser_pid, __ATOMIC_ACQUIRE);
		const uint32_t seq = __atomic_load_n(&h->release_seq, __ATOMIC_ACQUIRE);
		if (who != 0 && who != (int32_t)getpid()) {
			for (;;) {
				who = __atomic_load_n(&h->releaser_pid, __ATOMIC_ACQUIRE);
				if (who == 0 || __atomic_load_n(&h->release_seq, __ATOMIC_ACQUIRE) != seq ||
				    __atomic_load_n(&h->released_bytes, __ATOMIC_ACQUIRE) >= cap + slack)
					break;
				if (now_ms() - t0 > 2000.0 || (kill(who, 0) != 0 && errno == ESRCH))
					break; /* stuck or gone: fall back to asking the driver */
				fetch_retire_completed(e, rep); /* the releaser may be waiting for the units of what has landed here */
				pthread_mutex_unlock(&e->mu);
				usleep(200);
				pthread_mutex_lock(&e->mu);
			}
			fetch_retire_completed(e, rep);
			if (e->d.MemGetInfo(&free_b, &total_b) != CUDA_SUCCESS || free_b >= one_batch) {
				rep->wait_ms += now_ms() - t0;
				return 0;
			}
			last_free = free_b;
			last_growth = now_ms();
		}
	}
	for (;;) {
		const double now = now_ms(), waited = now - t0;
		if (free_b > last_free)
			last_growth = now; /* the previous holder is handing HBM back right now */
		last_free = free_b;
		if (free_b >= cap + slack)
			break;
		if (free_b >= one_batch && polls > 0 && now - last_growth >= NVS_SETTLE_MS)
			break; /* room for a batch and the releaser has paused: our calls will not collide with its */
		if (waited > e->cfg.oom_wait_ms) {
			nvs_warn("engine: HBM still exhausted after %.0f ms", waited);
			rep->wait_ms += waited;
			return NVS_E_TIMEOUT;
		}
		if (e->cfg.pressure_cb && now - last_growth >= PRESSURE_AFTER_MS && waited >= next_pressure) {
			e->cfg.pressure_cb(e->cfg.pressure_user, remaining);
			next_pressure = waited + 1000;
		}
		fetch_retire_completed(e, rep);
		pthread_mutex_unlock(&e->mu);
		usleep(polls < 100 ? 1000 : 2000);
		pthread_mutex_lock(&e->mu);
		++polls;
		if (e->d.MemGetInfo(&free_b, &total_b) != CUDA_SUCCESS)
			break;
	}
	rep->wait_ms += now_ms() - t0;
	return 0;
}

/* A batch has landed in HBM: its backing units go back to the pool at once, so
 * that the client evicting right now (other process, shared pool) can reuse them. */
static int fetch_retire(nvs_engine *e, struct slot *s, nvs_xfer_report *rep)
{
	int rc = 0;
	if (s->busy) {
		float ms = 0;
		CK(e, e->d.EventSynchronize(s->done));
		if (rep && e->d.EventElapsedTime(&ms, s->begin, s->done) == CUDA_SUCCESS)
			rep->copy_ms += ms;
		for (uint32_t i = 0; i < s->n_chunks; ++i)
			backing_after_fetch(e, s->chunks[i]); /* kept (reclaimable) or given back at once */
	}
out:
	s->busy = 0;
	slot_reset(s);
	return rc;
}

int nvs_fetch_all(nvs_engine *e, nvs_xfer_report *rep_out)
{
	nvs_xfer_report rep;
	memset(&rep, 0, sizeof(rep));
	if (!e)
		return NVS_E_BAD_ARG;
	int rc = 0;
	double t_begin = now_ms();
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	e->epoch++;

	int started = 0, deferred = 0;
	unsigned batch_no = 0;
	struct alloc *a = e->head;
	uint32_t ci = 0;
	uint64_t remaining = e->st.swapped_bytes + e->st.unbacked_bytes;
	for (;;) {
		/* next batch of non-resident chunks, allocation order */
		struct slot *s = &e->slots[batch_no % N_SLOTS];
		if ((rc = fetch_retire(e, s, &rep)) != 0)
			goto out;
		if (remaining && (rc = wait_for_hbm_burst(e, remaining, &rep)) != 0)
			goto out;
		uint64_t batch = 0, copy_bytes = 0;
		double t0 = now_ms();
		while (a && batch < e->cfg.batch_bytes) {
			if (a->passthrough || ci >= a->n_chunks) {
				a = a->next;
				ci = 0;
				continue;
			}
			struct chunk *c = &a->chunks[ci];
			if (c->state == CH_RESIDENT) {
				++ci;
				continue;
			}
			if (s->n_chunks == s->cap_chunks || s->n_descs + c->bytes / SLAB > s->cap_descs ||
			    s->n_ce + c->bytes / SLAB > s->cap_ce || s->n_aux + c->bytes / SLAB > s->cap_aux)
				break;
			double w = 0;
			if ((deferred = chunk_map(e, c, &w)) != 0)
				break; /* what this batch has mapped so far still gets its data before we give up */
			rep.wait_ms += w;
			rep.chunks++;
			if (c->state == CH_SWAPPED) {
				const uint64_t moving = c->bytes - (uint64_t)c->n_const * SLAB;
				uint64_t want[MAX_CHUNK_SLABS / 64]; /* every slab that has bytes in the backing */
				mask_fill(want, (uint32_t)(c->bytes / SLAB));
				for (uint32_t k = 0; k < MAX_CHUNK_SLABS / 64; ++k)
					want[k] &= ~c->cmask[k];
				slot_push_chunk(e, s, c, 0, want);
				/* same-filled slabs are re-created on the device instead of copied */
				for (uint32_t k = 0; c->n_const && k < c->bytes / SLAB; ++k) {
					if (!slab_is_const(c, k) || s->n_aux == s->cap_aux)
						continue;
					nvs_copy_desc *d = &s->aux[s->n_aux++];
					d->src = c->cvals[k];
					d->dst = c->va + (uint64_t)k * SLAB;
					d->bytes = SLAB;
					d->tag = 0;
				}
				rep.elided_bytes += (uint64_t)c->n_const * SLAB;
				copy_bytes += moving;
				if (c->tier >= TIER_PEER0)
					rep.peer_bytes += moving;
				else
					rep.host_bytes += moving;
				memset(c->cmask, 0, sizeof(c->cmask));
				c->n_const = 0;
			} /* UNBACKED: map only, nothing to copy */
			c->epoch = e->epoch;
			state_account(e, c, CH_RESIDENT);
			batch += c->bytes;
			remaining = remaining > c->bytes ? remaining - c->bytes : 0;
			++ci;
		}
		rep.map_ms += now_ms() - t0;
		if (batch == 0) {
			if (a && !deferred) /* a chunk that cannot fit an empty slot: geometry bug */
				rc = NVS_E_BAD_ARG;
			break;
		}
		if (s->n_descs || s->n_ce || s->n_aux) {
			started = 1;
			CK(e, e->d.EventRecord(s->begin, e->stream));
			if ((rc = slot_launch(e, s, kernel_variant(e, 0), &rep)) != 0)
				goto out;
			if ((rc = launch_aux(e, e->fn_splat, s, e->stream, 0, 0)) != 0)
				goto out;
			CK(e, e->d.EventRecord(s->done, e->stream));
			s->busy = 1;
			rep.launches += s->n_aux ? 1 : 0;
			rep.bytes += copy_bytes;
			rep.slabs += copy_bytes / SLAB;
		}
		batch_no++;
		if (deferred)
			break;
	}
	(void)started;
	for (unsigned k = 0; k < N_SLOTS; ++k)
		if ((rc = fetch_retire(e, &e->slots[k], &rep)) != 0)
			goto out;
	if (deferred) {
		/* every chunk marked resident holds its data; the rest is still swapped out */
		rc = deferred;
		goto out;
	}
	e->resident_mode = 1;
	e->st.n_fetches++;
	e->st.fetched_bytes_total += rep.bytes;
out:
	if (rc != 0 && e->d.StreamSynchronize(e->stream) == CUDA_SUCCESS) {
		/* batches already launched have landed: their backing is no longer needed */
		for (unsigned k = 0; k < N_SLOTS; ++k)
			for (uint32_t i = 0; e->slots[k].busy && i < e->slots[k].n_chunks; ++i)
				backing_after_fetch(e, e->slots[k].chunks[i]);
	}
	for (unsigned k = 0; k < N_SLOTS; ++k) {
		e->slots[k].busy = 0;
		slot_reset(&e->slots[k]);
	}
	rep.map_ms -= rep.wait_ms;
	if (rep.map_ms < 0)
		rep.map_ms = 0;
	rep.wall_ms = now_ms() - t_begin;
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	if (rc == 0 && (rep.bytes || rep.chunks || rep.elided_bytes))
		report_emit(e, "fetch", &rep, 0);
	if (rep_out)
		*rep_out = rep;
	return rc;
}

/* ---------------------------------------------------------- pre-clean ---- */

/*
 * SURVEY 8f rank 3, first half: while the owner of the lock computes, the link to the backing
 * tier is idle.  This thread uses it: one resident chunk at a time that has no (complete)
 * backing copy is written back by the FUSED copy + hash kernel (nvs_slab_scan with a
 * destination) on a lowest-priority stream with a handful of CTAs.  Every lane hashes exactly
 * the vectors it stores, so the recorded hashes describe the bytes in the backing copy whatever
 * the application's kernels were doing to the source meanwhile; at the hand-off the eviction
 * scan compares them with the hashes of the then-current contents and copies only what differs.
 * A chunk that keeps turning out dirty is left alone (ST_VOLATILE, re-probed now and then); only
 * FREE pool units are used, and the copies are the first thing anybody short of units takes
 * over (RS_PLAIN).  The reference has no counterpart: UVM pages stay put until somebody faults.
 */
static struct chunk *preclean_pick(nvs_engine *e)
{
	for (struct alloc *a = e->head; a; a = a->next) {
		if (a->passthrough)
			continue;
		for (uint32_t i = 0; i < a->n_chunks; ++i) {
			struct chunk *c = &a->chunks[i];
			if (c->state != CH_RESIDENT || c->backing || c->scanned)
				continue;
			if (c->stable == ST_VOLATILE) { /* was dirty against its copy last time: mostly not worth it */
				if (c->volatile_skips < VOLATILE_REPROBE)
					continue;
			}
			if (c->pre_epoch == e->epoch + 1)
				continue; /* already tried during this residency */
			return c;
		}
	}
	return NULL;
}

static void *preclean_main(void *arg)
{
	nvs_engine *e = arg;
	sigset_t all; /* this thread lives inside an arbitrary application */
	sigfillset(&all);
	pthread_sigmask(SIG_SETMASK, &all, NULL);
	if (ctx_enter(e) != 0)
		return NULL;
	uint64_t pass_bytes = 0;
	pthread_mutex_lock(&e->mu);
	while (!e->stopping) {
		if (!e->resident_mode) {
			pthread_cond_wait(&e->pre_cv, &e->mu);
			continue;
		}
		pthread_mutex_unlock(&e->mu);
		/* api_mu keeps evict / fetch / free away from the chunk while its copy is in flight */
		pthread_mutex_lock(&e->api_mu);
		pthread_mutex_lock(&e->mu);
		struct chunk *c = (e->resident_mode && !e->stopping) ? preclean_pick(e) : NULL;
		int launched = 0;
		if (c) {
			c->pre_epoch = e->epoch + 1;
			const uint32_t n = (uint32_t)(c->bytes / SLAB);
			const uint32_t tag = ++e->tag_next ? e->tag_next : ++e->tag_next;
			/* free units only: never take over anybody's kept copy, never wait, never pin inline */
			if (pool_take(e, &e->host_pool, n, &c->backing, 0, tag) == 0) {
				c->tier = TIER_HOST;
				c->btag = tag;
				e->st.host_pool_used = e->host_pool.used;
				for (uint32_t k = 0; k < n; ++k) {
					e->pre_descs[k].src = c->va + (uint64_t)k * SLAB;
					e->pre_descs[k].dst = c->backing + (uint64_t)k * SLAB;
					e->pre_descs[k].bytes = SLAB;
					e->pre_descs[k].tag = 0;
				}
				uint32_t nn = n, want_hash = 1;
				unsigned grid = n < 8 ? n : 8;
				void *params[] = {&e->pre_descs_dev, &nn, &e->pre_counter, &e->pre_out_dev, &want_hash};
				if (e->d.MemsetD32Async(e->pre_counter, 0, 1, e->pre_stream) == CUDA_SUCCESS &&
				    e->d.LaunchKernel(e->fn_scan, grid, 1, 1, 256, 1, 1, 0, e->pre_stream, params, NULL) == CUDA_SUCCESS &&
				    e->d.EventRecord(e->pre_done, e->pre_stream) == CUDA_SUCCESS) {
					launched = 1;
					e->st.kernel_launches_total++;
				} else {
					pool_give(e, &e->host_pool, c->backing, n, c->btag);
					c->backing = 0;
					c->tier = TIER_NONE;
				}
			} else if (e->shp && e->cfg.prepin && e->host_pool.bytes < (uint64_t)e->shp->n_windows * e->cfg.host_arena_bytes) {
				/* let the pinning thread bring the next window in; try again on the next round */
				c->pre_epoch = 0;
				e->pin_target = e->host_pool.bytes + e->cfg.host_arena_bytes;
				pthread_cond_signal(&e->pin_cv);
			} else if (!e->shp && e->cfg.prepin && e->host_pool.bytes < e->pin_target) {
				/* private pool: the pinning thread is still on its way to the footprint; same */
				c->pre_epoch = 0;
			}
		}
		if (launched) {
			pthread_mutex_unlock(&e->mu);
			CUresult r = e->d.EventSynchronize(e->pre_done);
			pthread_mutex_lock(&e->mu);
			const uint32_t n = (uint32_t)(c->bytes / SLAB);
			if (r == CUDA_SUCCESS && (c->hash || (c->hash = malloc(MAX_CHUNK_SLABS * sizeof(struct slab_hash))))) {
				for (uint32_t k = 0; k < n; ++k) {
					c->hash[k].h0 = e->pre_out[k].h0;
					c->hash[k].h1 = e->pre_out[k].h1;
				}
				mask_fill(c->bvalid, n); /* the copy holds bytes for every slab, same-filled or not */
				backing_mark_retained(e, c);
				e->st.precleaned_bytes_total += c->bytes;
				pass_bytes += c->bytes;
			} else {
				pool_give(e, &e->host_pool, c->backing, n, c->btag);
				c->backing = 0;
				c->tier = TIER_NONE;
			}
			e->st.host_pool_used = e->host_pool.used;
		}
		const int more = c != NULL;
		if (!more && pass_bytes) {
			if (e->stats_file) {
				fprintf(e->stats_file, "{\"op\":\"preclean\",\"t\":%.6f,\"pid\":%d,\"bytes\":%" PRIu64 ",\"retained_bytes\":%" PRIu64
					",\"pool_used\":%" PRIu64 "}\n", wall_s(), (int)getpid(), pass_bytes, e->st.retained_bytes, e->host_pool.used);
				fflush(e->stats_file);
			}
			nvs_debug("engine: pre-cleaned %" PRIu64 " MiB in the background", pass_bytes >> 20);
			pass_bytes = 0;
		}
		pthread_mutex_unlock(&e->mu);
		pthread_mutex_unlock(&e->api_mu);
		if (more) {
			usleep(1000); /* leave the entry points room between two chunks */
			pthread_mutex_lock(&e->mu);
		} else {
			/* nothing to do right now: sleep until the next lock grant (or for a while: new allocations) */
			struct timespec until;
			clock_gettime(CLOCK_REALTIME, &until);
			until.tv_sec += 1;
			pthread_mutex_lock(&e->mu);
			if (!e->stopping)
				pthread_cond_timedwait(&e->pre_cv, &e->mu, &until);
		}
	}
	pthread_mutex_unlock(&e->mu);
	ctx_leave(e);
	return NULL;
}

/* ------------------------------------------------------ alloc / free ---- */

void nvs_set_resident_mode(nvs_engine *e, int holds_lock)
{
	if (!e)
		return;
	pthread_mutex_lock(&e->mu);
	e->resident_mode = holds_lock != 0;
	if (e->resident_mode && e->pre_thread_started)
		pthread_cond_signal(&e->pre_cv);
	pthread_mutex_unlock(&e->mu);
}

int nvs_alloc(nvs_engine *e, uint64_t *dptr, uint64_t bytes)
{
	if (!e || !dptr)
		return NVS_E_BAD_ARG;
	if (bytes == 0)
		return CUDA_ERROR_INVALID_VALUE;
	int rc = 0;
	struct alloc *a = calloc(1, sizeof(*a));
	if (!a)
		return CUDA_ERROR_OUT_OF_MEMORY;
	if (ctx_enter(e) != 0) {
		free(a);
		return CUDA_ERROR_INVALID_CONTEXT;
	}
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	a->req_bytes = bytes;

	if (bytes < e->cfg.small_alloc_bytes) {
		/* not worth a 2 MiB granule: stays ordinary (always resident) device memory */
		CUdeviceptr p = 0;
		CUresult r = e->d.MemAlloc(&p, bytes);
		if (r != CUDA_SUCCESS) {
			rc = (int)r;
			goto out;
		}
		a->va = p;
		a->va_bytes = bytes;
		a->passthrough = 1;
		e->st.passthrough_bytes += bytes;
		table_insert(e, a);
		*dptr = p;
		a = NULL;
		goto out;
	}

	a->va_bytes = (bytes + SLAB - 1) & ~(SLAB - 1);
	a->n_chunks = (uint32_t)((a->va_bytes + e->cfg.chunk_bytes - 1) / e->cfg.chunk_bytes);
	a->chunks = calloc(a->n_chunks, sizeof(struct chunk));
	if (!a->chunks) {
		rc = CUDA_ERROR_OUT_OF_MEMORY;
		goto out;
	}
	CUdeviceptr va = 0;
	CUresult r = e->d.MemAddressReserve(&va, a->va_bytes, 0, 0, 0);
	if (r != CUDA_SUCCESS) {
		rc = (int)r;
		goto out;
	}
	a->va = va;
	for (uint32_t i = 0; i < a->n_chunks; ++i) {
		struct chunk *c = &a->chunks[i];
		c->va = va + (uint64_t)i * e->cfg.chunk_bytes;
		uint64_t left = a->va_bytes - (uint64_t)i * e->cfg.chunk_bytes;
		c->bytes = left < e->cfg.chunk_bytes ? left : e->cfg.chunk_bytes;
		c->owner = a;
		c->state = CH_UNBACKED;
		e->st.unbacked_bytes += c->bytes;
	}
	if (e->resident_mode) {
		for (uint32_t i = 0; i < a->n_chunks; ++i) {
			struct chunk *c = &a->chunks[i];
			if ((rc = chunk_map_ex(e, c, NULL, 1)) == NVS_I_LOCK_LOST) {
				/* the quantum ended while we were waiting for HBM: what is mapped stays, the rest of
				 * the allocation is virtual until this client is granted the lock again (nvs_fetch_all) */
				rc = 0;
				break;
			}
			if (rc != 0) {
				for (uint32_t k = 0; k < i; ++k) {
					chunk_unmap(e, &a->chunks[k]);
					state_account(e, &a->chunks[k], CH_UNBACKED);
				}
				for (uint32_t k = 0; k < a->n_chunks; ++k)
					e->st.unbacked_bytes -= a->chunks[k].bytes;
				e->d.MemAddressFree(va, a->va_bytes);
				if (rc == NVS_E_TIMEOUT)
					rc = CUDA_ERROR_OUT_OF_MEMORY;
				goto out;
			}
			c->epoch = e->epoch;
			state_account(e, c, CH_RESIDENT);
		}
	}
	e->st.va_bytes += a->va_bytes;
	nvs_gl_own(e->gl_dev, (int64_t)a->va_bytes); /* what this process needs resident here when it holds the lock */
	table_insert(e, a);
	*dptr = va;
	/* keep the pinned pool ahead of what may have to be swapped out (private pool:
	 * the whole footprint; shared pool: a head start, the rest follows the usage) */
	if (e->cfg.prepin && e->cfg.n_peers == 0) {
		if (!e->shp)
			e->pin_target += a->va_bytes;
		else if (e->pin_target < 8 * e->cfg.host_arena_bytes)
			e->pin_target = 8 * e->cfg.host_arena_bytes;
		pthread_cond_signal(&e->pin_cv);
	}
	a = NULL;
out:
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	if (a) {
		free(a->chunks);
		free(a);
	}
	return rc;
}

int nvs_free(nvs_engine *e, uint64_t dptr)
{
	return nvs_free_sized(e, dptr, NULL);
}

int nvs_free_sized(nvs_engine *e, uint64_t dptr, uint64_t *req_bytes)
{
	if (!e)
		return NVS_E_BAD_ARG;
	int rc = 0;
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	struct alloc *a = table_find(e, dptr);
	if (!a) {
		rc = NVS_E_NOT_OURS;
		goto out;
	}
	if (req_bytes)
		*req_bytes = a->req_bytes;
	if (a->passthrough) {
		CUresult r = e->d.MemFree(a->va);
		if (r != CUDA_SUCCESS) {
			rc = (int)r;
			goto out;
		}
		e->st.passthrough_bytes -= a->req_bytes;
	} else {
		/* cuMemFree synchronises implicitly (which is what the reference's hook ends up calling,
		 * src/hook.c:691); cuMemUnmap / cuMemRelease are not documented to.  Work of the application
		 * that is still in flight must not find its pages gone -- or handed to another client. */
		for (uint32_t i = 0; i < a->n_chunks; ++i)
			if (a->chunks[i].state == CH_RESIDENT) {
				CUresult r = e->d.CtxSynchronize();
				if (r != CUDA_SUCCESS && !is_shutdown_error(r))
					nvs_warn("engine: cuCtxSynchronize before unmapping returned %s", cu_name(e, r));
				break;
			}
		for (uint32_t i = 0; i < a->n_chunks; ++i) {
			struct chunk *c = &a->chunks[i];
			if (c->state == CH_RESIDENT)
				chunk_unmap(e, c);
			backing_release(e, c);
			free(c->cvals);
			free(c->hash);
			free(c->nh);
			c->cvals = NULL;
			c->hash = c->nh = NULL;
			uint64_t *ctr = c->state == CH_RESIDENT ? &e->st.resident_bytes
					: c->state == CH_SWAPPED ? &e->st.swapped_bytes
								 : &e->st.unbacked_bytes;
			*ctr -= c->bytes;
		}
		e->d.MemAddressFree(a->va, a->va_bytes);
		e->st.va_bytes -= a->va_bytes;
		nvs_gl_own(e->gl_dev, -(int64_t)a->va_bytes);
		if (e->cfg.prepin && e->cfg.n_peers == 0 && !e->shp && e->pin_target >= a->va_bytes)
			e->pin_target -= a->va_bytes;
	}
	table_remove(e, a);
	free(a->chunks);
	free(a);
out:
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	return rc;
}

/* ------------------------------------------- lock-free host<->backing ---- */

static struct alloc *table_find_range(nvs_engine *e, uint64_t addr, uint64_t bytes)
{
	const size_t at = by_va_upper(e, addr);
	if (at == 0)
		return NULL;
	struct alloc *a = e->by_va[at - 1];
	if (addr - a->va < a->va_bytes)
		return bytes <= a->va_bytes - (addr - a->va) ? a : NULL;
	return NULL;
}

/* host address of a host-tier chunk's backing copy; e->mu held */
static uint8_t *backing_host_ptr(nvs_engine *e, const struct chunk *c)
{
	for (struct arena *ar = e->host_pool.arenas; ar; ar = ar->next)
		if (c->backing >= ar->dev_base && c->backing < ar->dev_base + ar->bytes)
			return (uint8_t *)ar->host_base + (c->backing - ar->dev_base);
	return NULL;
}

static void fill_words(uint8_t *dst, uint64_t slab_off, uint64_t n, uint64_t value)
{
	/* the slab is `value` repeated from its first byte on: byte k is byte (k & 7) of value */
	const uint8_t *v = (const uint8_t *)&value;
	uint64_t k = 0;
	for (; k < n && ((slab_off + k) & 7); ++k)
		dst[k] = v[(slab_off + k) & 7];
	for (; k + 8 <= n; k += 8)
		memcpy(dst + k, &value, 8);
	for (; k < n; ++k)
		dst[k] = v[(slab_off + k) & 7];
}

/* Large copies are split over a few threads: one core moves ~6 GB/s, the DRAM several times that. */
struct memcpy_job {
	uint8_t *dst;
	const uint8_t *src;
	size_t n;
};

static void *memcpy_worker(void *arg)
{
	struct memcpy_job *j = arg;
	memcpy(j->dst, j->src, j->n);
	return NULL;
}

static void par_memcpy(uint8_t *dst, const uint8_t *src, uint64_t n)
{
	enum { MAX_T = 6 };
	const uint64_t piece_min = 16ull << 20;
	unsigned t = (unsigned)(n / piece_min);
	if (t > MAX_T)
		t = MAX_T;
	if (t < 2) {
		memcpy(dst, src, n);
		return;
	}
	pthread_t th[MAX_T];
	struct memcpy_job jobs[MAX_T];
	const uint64_t piece = (n / t + 4095) & ~4095ull;
	unsigned started = 0;
	uint64_t off = 0;
	sigset_t all, old; /* the helpers must never run the application's signal handlers */
	sigfillset(&all);
	pthread_sigmask(SIG_BLOCK, &all, &old);
	for (unsigned i = 0; i + 1 < t && off + piece < n; ++i, off += piece) {
		jobs[i] = (struct memcpy_job){dst + off, src + off, piece};
		if (pthread_create(&th[i], NULL, memcpy_worker, &jobs[i]) != 0)
			break;
		started++;
	}
	pthread_sigmask(SIG_SETMASK, &old, NULL);
	off = (uint64_t)started * piece;
	memcpy(dst + off, src + off, n - off); /* the calling thread takes the rest */
	for (unsigned i = 0; i < started; ++i)
		pthread_join(th[i], NULL);
}

int nvs_host_io(nvs_engine *e, uint64_t dptr, void *host, uint64_t bytes, int to_device)
{
	if (!e || !host || bytes == 0)
		return NVS_E_BAD_ARG;
	int rc = 0;
	/* api_mu keeps evict / fetch / free away for the whole call; mu is only taken
	 * where the pools are consulted, never across a memcpy */
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	struct alloc *a = table_find_range(e, dptr, bytes);
	if (!a || a->passthrough) {
		rc = NVS_E_NOT_OURS;
		goto out;
	}
	const uint64_t off0 = dptr - a->va;
	const uint32_t first = (uint32_t)(off0 / e->cfg.chunk_bytes);
	const uint32_t last = (uint32_t)((off0 + bytes - 1) / e->cfg.chunk_bytes);
	for (uint32_t ci = first; ci <= last; ++ci) {
		const struct chunk *c = &a->chunks[ci];
		if (c->state == CH_RESIDENT || (c->backing && c->tier != TIER_HOST) ||
		    (c->state == CH_UNBACKED && (!to_device || e->cfg.n_peers > 0)) ||
		    (!c->backing && e->cfg.n_peers > 0)) {
			rc = NVS_E_NOT_SWAPPED;
			goto out;
		}
	}
	uint8_t *h = host;
	for (uint32_t ci = first; ci <= last; ++ci) {
		struct chunk *c = &a->chunks[ci];
		const uint64_t c_off = (uint64_t)ci * e->cfg.chunk_bytes;
		const uint64_t lo = off0 > c_off ? off0 - c_off : 0;
		const uint64_t hi = off0 + bytes - c_off < c->bytes ? off0 + bytes - c_off : c->bytes;
		if (to_device && !c->backing) {
			/* never materialised, or every slab same-filled: it needs a backing copy now */
			int need_ctx = ctx_enter(e) == 0; /* pinning a new arena needs the context */
			rc = backing_assign(e, c, 0);
			if (need_ctx)
				ctx_leave(e);
			if (rc != 0)
				goto out;
			if (c->state == CH_UNBACKED) {
				/* Untouched slabs become "same-filled with 0": the pool's pages may hold
				 * another client's old data, which must neither be copied nor leak. */
				const uint32_t n_slabs = (uint32_t)(c->bytes / SLAB);
				if (!c->cvals && !(c->cvals = calloc(MAX_CHUNK_SLABS, sizeof(uint64_t)))) {
					backing_release(e, c);
					rc = NVS_E_HOST_OOM;
					goto out;
				}
				memset(c->cvals, 0, MAX_CHUNK_SLABS * sizeof(uint64_t));
				for (uint32_t k = 0; k < n_slabs; ++k)
					c->cmask[k >> 6] |= 1ull << (k & 63);
				c->n_const = n_slabs;
				state_account(e, c, CH_SWAPPED);
			}
		}
		uint8_t *b = c->backing ? backing_host_ptr(e, c) : NULL;
		if (c->backing && !b) {
			rc = NVS_E_NOT_SWAPPED;
			goto out;
		}
		pthread_mutex_unlock(&e->mu);
		for (uint64_t at = lo; at < hi;) {
			const uint32_t si = (uint32_t)(at / SLAB);
			uint64_t s_end = ((uint64_t)si + 1) * SLAB < hi ? ((uint64_t)si + 1) * SLAB : hi;
			if (slab_is_const(c, si) && !to_device) {
				fill_words(h, at - (uint64_t)si * SLAB, s_end - at, c->cvals[si]);
				h += s_end - at;
				at = s_end;
				continue;
			}
			/* one copy for a whole run of slabs that have (or now get) real bytes in the backing */
			for (uint32_t k = si;; ++k) {
				if (slab_is_const(c, k)) {
					if (!to_device)
						break;
					/* stops being same-filled: unless it is overwritten entirely, write it out first */
					const uint64_t k_lo = (uint64_t)k * SLAB, k_hi = k_lo + SLAB;
					if (at > k_lo || hi < k_hi)
						fill_words(b + k_lo, 0, SLAB, c->cvals[k]);
					c->cmask[k >> 6] &= ~(1ull << (k & 63));
					c->n_const--;
				}
				s_end = ((uint64_t)k + 1) * SLAB < hi ? ((uint64_t)k + 1) * SLAB : hi;
				if (s_end == hi)
					break;
			}
			if (to_device) {
				/* the backing copy changes under its recorded hashes: they no longer describe it */
				for (uint32_t k = (uint32_t)(at / SLAB); (uint64_t)k * SLAB < s_end; ++k)
					c->bvalid[k >> 6] &= ~(1ull << (k & 63));
				par_memcpy(b + at, h, s_end - at);
			} else
				par_memcpy(h, b + at, s_end - at);
			h += s_end - at;
			at = s_end;
		}
		pthread_mutex_lock(&e->mu);
	}
	e->st.host_io_bytes_total += bytes;
out:
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	return rc;
}

int nvs_lookup(nvs_engine *e, uint64_t dptr, uint64_t *req_bytes)
{
	if (!e)
		return NVS_E_BAD_ARG;
	pthread_mutex_lock(&e->mu);
	struct alloc *a = table_find(e, dptr);
	if (a && req_bytes)
		*req_bytes = a->req_bytes;
	pthread_mutex_unlock(&e->mu);
	return a ? 0 : NVS_E_NOT_OURS;
}

int nvs_touch(nvs_engine *e, uint64_t dptr, uint64_t bytes)
{
	if (!e || bytes == 0)
		return NVS_E_BAD_ARG;
	int rc = NVS_E_NOT_OURS;
	pthread_mutex_lock(&e->mu);
	struct alloc *a = table_find_range(e, dptr, bytes);
	if (a && !a->passthrough) {
		const uint64_t off0 = dptr - a->va, now = ++e->touch_clock;
		for (uint32_t ci = (uint32_t)(off0 / e->cfg.chunk_bytes); ci <= (uint32_t)((off0 + bytes - 1) / e->cfg.chunk_bytes); ++ci)
			a->chunks[ci].touch = now;
		rc = 0;
	}
	pthread_mutex_unlock(&e->mu);
	return rc;
}

int nvs_get_stats(nvs_engine *e, nvs_stats *out)
{
	if (!e || !out)
		return NVS_E_BAD_ARG;
	pthread_mutex_lock(&e->mu);
	e->st.host_pool_bytes = e->host_pool.bytes;
	e->st.host_pool_used = e->host_pool.used;
	*out = e->st;
	pthread_mutex_unlock(&e->mu);
	return 0;
}

/* ------------------------------------------------- raw kernel access ---- */

int nvs_copy_slabs(nvs_engine *e, const nvs_copy_desc *descs, uint32_t n, uint32_t variant, uint32_t grid,
		   float *ms_out)
{
	if (!e || (!descs && n))
		return NVS_E_BAD_ARG;
	for (uint32_t i = 0; i < n; ++i) {
		if ((descs[i].src | descs[i].dst) & 15ull)
			return NVS_E_BAD_ARG;
		if (variant == NVS_COPY_TMA && (descs[i].bytes & 15ull))
			return NVS_E_BAD_ARG;
	}
	int rc = 0;
	void *staging = NULL;
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	const size_t bytes = (size_t)n * sizeof(nvs_copy_desc);
	CUdeviceptr dev = 0;
	if (n) {
		CK(e, e->d.MemHostAlloc(&staging, bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
		memcpy(staging, descs, bytes);
		if (e->d.MemHostGetDevicePointer(&dev, staging, 0) != CUDA_SUCCESS)
			dev = (CUdeviceptr)(uintptr_t)staging;
	}
	CK(e, e->d.EventRecord(e->ev_begin, e->stream));
	if ((rc = launch_descs(e, dev, staging, n, variant, grid_for(e, grid, 0))) != 0)
		goto out;
	CK(e, e->d.EventRecord(e->ev_end, e->stream));
	CK(e, e->d.EventSynchronize(e->ev_end));
	if (ms_out)
		CK(e, e->d.EventElapsedTime(ms_out, e->ev_begin, e->ev_end));
out:
	if (rc != 0)
		e->d.StreamSynchronize(e->stream);
	if (staging)
		e->d.MemFreeHost(staging);
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	return rc;
}

int nvs_scan_slabs(nvs_engine *e, const nvs_copy_desc *descs, uint32_t n, int want_hash, nvs_scan_out *out, float *ms_out)
{
	if (!e || (!descs && n) || (!out && n))
		return NVS_E_BAD_ARG;
	for (uint32_t i = 0; i < n; ++i)
		if ((descs[i].src & 15ull) || (descs[i].bytes & 15ull) || descs[i].bytes == 0)
			return NVS_E_BAD_ARG;
	if (n == 0)
		return 0;
	int rc = 0;
	void *staging = NULL;
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	const size_t in_bytes = (size_t)n * sizeof(nvs_copy_desc), out_bytes = (size_t)n * sizeof(struct scan_result);
	CUdeviceptr dev = 0;
	CK(e, e->d.MemHostAlloc(&staging, in_bytes + out_bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	memcpy(staging, descs, in_bytes);
	if (e->d.MemHostGetDevicePointer(&dev, staging, 0) != CUDA_SUCCESS)
		dev = (CUdeviceptr)(uintptr_t)staging;
	{
		/* a private counter: this entry point may be handed any number of descriptors */
		CUdeviceptr counter = e->scratch + 16, out_dev = dev + in_bytes;
		uint32_t nn = n, wh = want_hash ? 1u : 0u;
		unsigned grid = n < (unsigned)e->n_sms * 4u ? n : (unsigned)e->n_sms * 4u;
		void *params[] = {&dev, &nn, &counter, &out_dev, &wh};
		CK(e, e->d.MemsetD32Async(counter, 0, 1, e->stream));
		CK(e, e->d.EventRecord(e->ev_begin, e->stream));
		CK(e, e->d.LaunchKernel(e->fn_scan, grid, 1, 1, 256, 1, 1, 0, e->stream, params, NULL));
		CK(e, e->d.EventRecord(e->ev_end, e->stream));
		CK(e, e->d.EventSynchronize(e->ev_end));
		e->st.kernel_launches_total++;
		if (ms_out)
			CK(e, e->d.EventElapsedTime(ms_out, e->ev_begin, e->ev_end));
		memcpy(out, (char *)staging + in_bytes, out_bytes);
	}
out:
	if (rc != 0)
		e->d.StreamSynchronize(e->stream);
	if (staging)
		e->d.MemFreeHost(staging);
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	return rc;
}

int nvs_pattern_fill(nvs_engine *e, uint64_t addr, uint64_t n_words, uint64_t first_index, uint64_t seed)
{
	if (!e || (addr & 7))
		return NVS_E_BAD_ARG;
	int rc = 0;
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	void *params[] = {&addr, &n_words, &first_index, &seed};
	CK(e, e->d.LaunchKernel(e->fn_fill, (unsigned)e->n_sms * 8, 1, 1, 256, 1, 1, 0, e->stream, params, NULL));
	CK(e, e->d.StreamSynchronize(e->stream));
out:
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	return rc;
}

int nvs_pattern_verify(nvs_engine *e, uint64_t addr, uint64_t n_words, uint64_t first_index, uint64_t seed,
		       uint64_t *mismatches)
{
	if (!e || (addr & 7) || !mismatches)
		return NVS_E_BAD_ARG;
	int rc = 0;
	if (ctx_enter(e) != 0)
		return CTX_GONE;
	pthread_mutex_lock(&e->api_mu);
	pthread_mutex_lock(&e->mu);
	CUdeviceptr out = e->scratch;
	uint64_t *host = NULL;
	CK(e, e->d.MemHostAlloc((void **)&host, 8, CU_MEMHOSTALLOC_PORTABLE));
	CK(e, e->d.MemsetD32Async(out, 0, 2, e->stream));
	void *params[] = {&addr, &n_words, &first_index, &seed, &out};
	CK(e, e->d.LaunchKernel(e->fn_verify, (unsigned)e->n_sms * 8, 1, 1, 256, 1, 1, 0, e->stream, params, NULL));
	CK(e, e->d.MemcpyAsync((CUdeviceptr)(uintptr_t)host, out, 8, e->stream));
	CK(e, e->d.StreamSynchronize(e->stream));
	*mismatches = *host;
out:
	if (host)
		e->d.MemFreeHost(host);
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&e->api_mu);
	ctx_leave(e);
	return rc;
}

/* ---------------------------------------------------- create/destroy ---- */

static void slots_free(nvs_engine *e)
{
	for (unsigned k = 0; k < N_SLOTS; ++k) {
		struct slot *s = &e->slots[k];
		if (s->descs)
			e->d.MemFreeHost(s->descs);
		if (s->aux)
			e->d.MemFreeHost(s->aux);
		if (s->scan_out)
			e->d.MemFreeHost(s->scan_out);
		if (s->done)
			e->d.EventDestroy(s->done);
		if (s->begin)
			e->d.EventDestroy(s->begin);
		free(s->chunks);
		free(s->ce);
		memset(s, 0, sizeof(*s));
	}
}

int nvs_engine_create(const nvs_engine_config *cfg_in, nvs_engine **out)
{
	if (!out)
		return NVS_E_BAD_ARG;
	*out = NULL;
	nvs_engine *e = calloc(1, sizeof(*e));
	if (!e)
		return CUDA_ERROR_OUT_OF_MEMORY;
	int rc = 0;
	int ctx_pushed = 0;
	e->gl_dev = e->host_pool.gl_dev = -1;
	for (int i = 0; i < NVS_MAX_PEERS; ++i)
		e->peer_pools[i].gl_dev = -1;
	if (cfg_in && cfg_in->struct_size == sizeof(e->cfg))
		e->cfg = *cfg_in;
	else if (cfg_in)
		{ free(e); return NVS_E_BAD_ARG; }
	else
		nvs_engine_default_config(&e->cfg);
	if (getenv("NVSHARE_DEBUG") && !nvs_debug_enabled) /* (inside the interposer hook.c has set it already: no store under the other threads' reads) */
		nvs_debug_enabled = 1;

	/* sanity of geometry */
	if (e->cfg.chunk_bytes < SLAB || (e->cfg.chunk_bytes & (SLAB - 1)) || e->cfg.chunk_bytes > MAX_CHUNK_SLABS * SLAB || e->cfg.host_arena_bytes < e->cfg.chunk_bytes ||
	    (e->cfg.host_arena_bytes & (SLAB - 1)) || e->cfg.tma_warps == 0 || e->cfg.tma_warps > 8 ||
	    e->cfg.tma_stages < 2 || e->cfg.tma_stages > 8 || (e->cfg.tma_tile_bytes & 15) || e->cfg.tma_tile_bytes == 0 ||
	    (uint64_t)e->cfg.tma_warps * e->cfg.tma_stages * e->cfg.tma_tile_bytes > 200u * 1024u ||
	    e->cfg.ldg_threads == 0 || e->cfg.ldg_threads > 1024 || (e->cfg.ldg_threads & 31) ||
	    e->cfg.n_peers < NVS_PEERS_AUTO || e->cfg.n_peers > NVS_MAX_PEERS) {
		free(e);
		return NVS_E_BAD_ARG;
	}
	if (e->cfg.evict_variant > NVS_COPY_CE || e->cfg.fetch_variant > NVS_COPY_CE ||
	    e->cfg.peer_evict_variant > NVS_COPY_CE || e->cfg.peer_fetch_variant > NVS_COPY_CE) {
		free(e);
		return NVS_E_BAD_ARG;
	}
	if (e->cfg.batch_bytes < e->cfg.chunk_bytes)
		e->cfg.batch_bytes = e->cfg.chunk_bytes;

	nvs_resolve_fn resolve = e->cfg.resolve ? e->cfg.resolve : default_resolve;
	for (size_t i = 0; i < sizeof(DRV_SYMS) / sizeof(DRV_SYMS[0]); ++i) {
		void *p = resolve(DRV_SYMS[i].name);
		if (!p) {
			nvs_warn("engine: driver entry point %s not found", DRV_SYMS[i].name);
			free(e);
			return NVS_E_NO_DRIVER;
		}
		memcpy((char *)&e->d + DRV_SYMS[i].off, &p, sizeof(p));
	}
	/* optional entry points (older drivers / the test double do without) */
	*(void **)&e->d.StreamCreateWithPriority = resolve("cuStreamCreateWithPriority");
	*(void **)&e->d.CtxGetStreamPriorityRange = resolve("cuCtxGetStreamPriorityRange");
	*(void **)&e->d.DeviceGetUuid = resolve("cuDeviceGetUuid_v2");
	if (!e->d.DeviceGetUuid)
		*(void **)&e->d.DeviceGetUuid = resolve("cuDeviceGetUuid");
	*(void **)&e->d.DeviceTotalMem = resolve("cuDeviceTotalMem_v2");
	*(void **)&e->d.DeviceGetCount = resolve("cuDeviceGetCount");
	pthread_mutex_init(&e->api_mu, NULL);
	pthread_mutex_init(&e->mu, NULL);
	pthread_cond_init(&e->pre_cv, NULL);
	pthread_cond_init(&e->pin_cv, NULL);
	pthread_cond_init(&e->grow_cv, NULL);

	CK(e, e->d.CtxGetCurrent(&e->ctx));
	if (!e->ctx) {
		rc = CUDA_ERROR_INVALID_CONTEXT;
		goto out;
	}
	CK(e, e->d.CtxPushCurrent(e->ctx));
	ctx_pushed = 1;
	CUdevice dev;
	CK(e, e->d.CtxGetDevice(&dev));
	e->device = e->cfg.device >= 0 ? e->cfg.device : (int)dev;
	CK(e, e->d.DeviceGetAttribute(&e->n_sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev));
	numa_init(e, dev, resolve);
	e->pool_grace_ms = (double)env_u64("NVSHARE_POOL_GRACE_MS", (uint64_t)POOL_FULL_GRACE_MS);

	if (e->d.ModuleLoadData(&e->module, nvs_slab_copy_cubin) != CUDA_SUCCESS ||
	    e->d.ModuleGetFunction(&e->fn_tma, e->module, "nvs_slab_copy_tma") != CUDA_SUCCESS ||
	    e->d.ModuleGetFunction(&e->fn_ldg, e->module, "nvs_slab_copy_ldg") != CUDA_SUCCESS ||
	    e->d.ModuleGetFunction(&e->fn_fill, e->module, "nvs_slab_fill") != CUDA_SUCCESS ||
	    e->d.ModuleGetFunction(&e->fn_verify, e->module, "nvs_slab_verify") != CUDA_SUCCESS ||
	    e->d.ModuleGetFunction(&e->fn_scan, e->module, "nvs_slab_scan") != CUDA_SUCCESS ||
	    e->d.ModuleGetFunction(&e->fn_splat, e->module, "nvs_slab_splat") != CUDA_SUCCESS) {
		nvs_warn("engine: the embedded sm_90a image could not be loaded on this device");
		rc = NVS_E_NO_KERNEL;
		goto out;
	}
	CK(e, e->d.FuncSetAttribute(e->fn_tma, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, 200 * 1024));
	CK(e, e->d.StreamCreate(&e->stream, CU_STREAM_NON_BLOCKING));
	CK(e, e->d.StreamCreate(&e->scan_stream, CU_STREAM_NON_BLOCKING));
	CK(e, e->d.EventCreate(&e->scan_done, CU_EVENT_DEFAULT));
	CK(e, e->d.EventCreate(&e->scan_begin, CU_EVENT_DEFAULT));
	CK(e, e->d.EventCreate(&e->ev_begin, CU_EVENT_DEFAULT));
	CK(e, e->d.EventCreate(&e->ev_end, CU_EVENT_DEFAULT));
	CK(e, e->d.MemAlloc(&e->counters, 4 * 2 * N_COUNTERS));
	CK(e, e->d.MemAlloc(&e->scratch, 64));
	CK(e, e->d.MemsetD32Async(e->counters, 0, 2 * N_COUNTERS, e->stream));
	CK(e, e->d.StreamSynchronize(e->stream));

	{
		/* one slot holds one batch: batch_bytes / SLAB descriptors (+ one chunk of slack) */
		uint32_t cap_descs = (uint32_t)((e->cfg.batch_bytes + e->cfg.chunk_bytes) / SLAB);
		/* the scan lists are longer: a partial eviction first scans everything resident, 4 batches per launch */
		uint32_t cap_aux = (uint32_t)((4 * e->cfg.batch_bytes + e->cfg.chunk_bytes) / SLAB);
		uint32_t cap_chunks = cap_aux; /* worst case: every chunk is a single slab */
		for (unsigned k = 0; k < N_SLOTS; ++k) {
			struct slot *s = &e->slots[k];
			s->ce = calloc(cap_descs, sizeof(nvs_copy_desc));
			s->cap_ce = cap_descs;
			if (!s->ce) {
				rc = CUDA_ERROR_OUT_OF_MEMORY;
				goto out;
			}
			CK(e, e->d.MemHostAlloc((void **)&s->descs, (size_t)cap_descs * sizeof(nvs_copy_desc),
						CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
			CUdeviceptr dp = 0;
			if (e->d.MemHostGetDevicePointer(&dp, s->descs, 0) != CUDA_SUCCESS)
				dp = (CUdeviceptr)(uintptr_t)s->descs;
			s->descs_dev = dp;
			s->cap_descs = cap_descs;
			CK(e, e->d.MemHostAlloc((void **)&s->aux, (size_t)cap_aux * sizeof(nvs_copy_desc),
						CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
			if (e->d.MemHostGetDevicePointer(&dp, s->aux, 0) != CUDA_SUCCESS)
				dp = (CUdeviceptr)(uintptr_t)s->aux;
			s->aux_dev = dp;
			s->cap_aux = cap_aux;
			CK(e, e->d.MemHostAlloc((void **)&s->scan_out, (size_t)cap_aux * sizeof(struct scan_result),
						CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
			if (e->d.MemHostGetDevicePointer(&dp, s->scan_out, 0) != CUDA_SUCCESS)
				dp = (CUdeviceptr)(uintptr_t)s->scan_out;
			s->scan_out_dev = dp;
			s->chunks = calloc(cap_chunks, sizeof(*s->chunks));
			s->cap_chunks = cap_chunks;
			if (!s->chunks) {
				rc = CUDA_ERROR_OUT_OF_MEMORY;
				goto out;
			}
			CK(e, e->d.EventCreate(&s->begin, CU_EVENT_DEFAULT));
			CK(e, e->d.EventCreate(&s->done, CU_EVENT_DEFAULT));
		}
	}

	e->host_pool.device = -1;
	e->host_pool.gl_dev = -1;
	if (e->cfg.shared_pool_path && *e->cfg.shared_pool_path) {
		size_t free_b = 0, total_b = 0;
		uint64_t cap = e->cfg.shared_pool_bytes;
		if (!cap && e->d.MemGetInfo(&free_b, &total_b) == CUDA_SUCCESS)
			cap = ((uint64_t)total_b + (1ull << 30) - 1) & ~((1ull << 30) - 1); /* one HBM's worth */
		if (shp_open(e, e->cfg.shared_pool_path, cap) != 0)
			nvs_warn("engine: cannot use the shared host pool %s (%s); using a private pinned pool",
				 e->cfg.shared_pool_path, strerror(errno));
	}
	if (e->cfg.n_peers == NVS_PEERS_AUTO) {
		/* every other GPU this process can see and this GPU can reach: with the GPU ledger such a
		 * GPU only lends what its own clients do not need, so "all of them" is a safe answer */
		int count = 0;
		e->cfg.n_peers = 0;
		if (e->d.DeviceGetCount && e->d.DeviceGetCount(&count) == CUDA_SUCCESS)
			for (int d = 0; d < count && e->cfg.n_peers < NVS_MAX_PEERS; ++d) {
				int can = 0;
				if (d != e->device && e->d.DeviceCanAccessPeer(&can, e->device, d) == CUDA_SUCCESS && can)
					e->cfg.peers[e->cfg.n_peers++] = d;
			}
		nvs_debug("engine: NVSHARE_PEERS=auto: %d peer GPU(s) of device %d can back its slabs", e->cfg.n_peers, e->device);
	}
	for (int i = 0; i < e->cfg.n_peers; ++i) {
		int can = 0;
		e->peer_pools[i].device = e->cfg.peers[i];
		e->peer_pools[i].capacity = e->cfg.peer_capacity_bytes;
		if (e->cfg.peers[i] == e->device ||
		    e->d.DeviceCanAccessPeer(&can, e->device, e->cfg.peers[i]) != CUDA_SUCCESS || !can) {
			nvs_warn("engine: device %d cannot be used as a peer backing tier from device %d",
				 e->cfg.peers[i], e->device);
			rc = NVS_E_BAD_ARG;
			goto out;
		}
	}
	/* cross-process accounting per GPU (gpu_ledger.h): the GPU we compute on and every peer we lend from */
	e->gl_reserve = env_u64("NVSHARE_GPU_RESERVE_MIB", 1536) << 20; /* the slice the reference hides too, src/hook.c:45 */
	e->gl_dev = gl_register(e, e->device, &e->gl_total);
	for (int i = 0; i < e->cfg.n_peers; ++i)
		e->peer_pools[i].gl_dev = gl_register(e, e->cfg.peers[i], NULL);
	if (e->cfg.stats_path && *e->cfg.stats_path)
		e->stats_file = fopen(e->cfg.stats_path, "a");
	if (e->cfg.prepin && e->cfg.n_peers == 0) {
		if (pthread_create(&e->pin_thread, NULL, pin_thread_main, e) == 0)
			e->pin_thread_started = 1;
	}
	if (e->cfg.preclean && e->cfg.retain && e->cfg.n_peers == 0) {
		int lo = 0, hi = 0;
		CUdeviceptr dp = 0;
		if (!(e->d.StreamCreateWithPriority && e->d.CtxGetStreamPriorityRange &&
		      e->d.CtxGetStreamPriorityRange(&lo, &hi) == CUDA_SUCCESS &&
		      e->d.StreamCreateWithPriority(&e->pre_stream, CU_STREAM_NON_BLOCKING, lo) == CUDA_SUCCESS))
			CK(e, e->d.StreamCreate(&e->pre_stream, CU_STREAM_NON_BLOCKING));
		CK(e, e->d.EventCreate(&e->pre_done, CU_EVENT_DISABLE_TIMING));
		CK(e, e->d.MemHostAlloc((void **)&e->pre_descs, MAX_CHUNK_SLABS * (sizeof(nvs_copy_desc) + sizeof(struct scan_result)),
					CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
		if (e->d.MemHostGetDevicePointer(&dp, e->pre_descs, 0) != CUDA_SUCCESS)
			dp = (CUdeviceptr)(uintptr_t)e->pre_descs;
		e->pre_descs_dev = dp;
		e->pre_out = (struct scan_result *)(e->pre_descs + MAX_CHUNK_SLABS);
		e->pre_out_dev = dp + MAX_CHUNK_SLABS * sizeof(nvs_copy_desc);
		e->pre_counter = e->scratch + 32;
		if (pthread_create(&e->pre_thread, NULL, preclean_main, e) == 0)
			e->pre_thread_started = 1;
	}
	nvs_debug("engine: ready on device %d (%d SMs): chunk %" PRIu64 " MiB, evict=%u fetch=%u, peers=%d",
		  e->device, e->n_sms, e->cfg.chunk_bytes >> 20, e->cfg.evict_variant, e->cfg.fetch_variant,
		  e->cfg.n_peers);
out:
	if (ctx_pushed)
		ctx_leave(e);
	if (rc != 0) {
		nvs_engine_destroy(e);
		return rc;
	}
	*out = e;
	return 0;
}

void nvs_engine_destroy(nvs_engine *e)
{
	if (!e)
		return;
	if (e->pin_thread_started || e->pre_thread_started) {
		pthread_mutex_lock(&e->mu);
		e->stopping = 1;
		pthread_cond_broadcast(&e->pin_cv);
		pthread_cond_broadcast(&e->pre_cv);
		pthread_mutex_unlock(&e->mu);
		if (e->pin_thread_started)
			pthread_join(e->pin_thread, NULL);
		if (e->pre_thread_started)
			pthread_join(e->pre_thread, NULL);
	}
	int have_ctx = e->ctx && e->d.CtxPushCurrent && ctx_enter(e) == 0;
	if (have_ctx) {
		if (e->stream)
			e->d.StreamSynchronize(e->stream);
		while (e->head) {
			struct alloc *a = e->head;
			if (nvs_free(e, a->va) != 0) { /* the driver refused: drop our record of it anyway */
				table_remove(e, a);
				free(a->chunks);
				free(a);
			}
		}
		if (e->shp)
			shp_close(e);
		for (struct arena *a = e->host_pool.arenas, *nx; a; a = nx) {
			nx = a->next;
			e->d.MemFreeHost(a->host_base);
			arena_free(a);
		}
		for (int i = 0; i < NVS_MAX_PEERS; ++i)
			for (struct arena *a = e->peer_pools[i].arenas, *nx; a; a = nx) {
				nx = a->next;
				e->d.MemUnmap(a->dev_base, a->bytes);
				e->d.MemAddressFree(a->dev_base, a->bytes);
				e->d.MemRelease(a->handle);
				nvs_gl_return(e->peer_pools[i].gl_dev, a->bytes);
				arena_free(a);
			}
		slots_free(e);
		if (e->counters)
			e->d.MemFree(e->counters);
		if (e->scratch)
			e->d.MemFree(e->scratch);
		if (e->ev_begin)
			e->d.EventDestroy(e->ev_begin);
		if (e->ev_end)
			e->d.EventDestroy(e->ev_end);
		if (e->stream)
			e->d.StreamDestroy(e->stream);
		if (e->scan_stream)
			e->d.StreamDestroy(e->scan_stream);
		if (e->scan_done)
			e->d.EventDestroy(e->scan_done);
		if (e->scan_begin)
			e->d.EventDestroy(e->scan_begin);
		if (e->pre_done)
			e->d.EventDestroy(e->pre_done);
		if (e->pre_stream)
			e->d.StreamDestroy(e->pre_stream);
		if (e->pre_descs)
			e->d.MemFreeHost(e->pre_descs);
		if (e->module)
			e->d.ModuleUnload(e->module);
		ctx_leave(e);
	} else {
		/* no context to tear the arenas down in: the driver takes them back with the process,
		 * the ledger must not keep counting them for as long as the process lives on */
		for (int i = 0; i < NVS_MAX_PEERS; ++i)
			nvs_gl_return(e->peer_pools[i].gl_dev, e->peer_pools[i].bytes);
	}
	/* allocations whose free the driver refused (or that had no context to be freed in) are no
	 * longer this engine's to claim */
	if (e->st.va_bytes)
		nvs_gl_own(e->gl_dev, -(int64_t)e->st.va_bytes);
	if (e->stats_file)
		fclose(e->stats_file);
	pthread_mutex_destroy(&e->mu);
	pthread_mutex_destroy(&e->api_mu);
	pthread_cond_destroy(&e->pin_cv);
	pthread_cond_destroy(&e->grow_cv);
	pthread_cond_destroy(&e->pre_cv);
	free(e->by_va);
	free(e);
}
