/*
 * hook.c -- libnvshare.so's LD_PRELOAD interposer.
 *
 * Drop-in boundary kept from the reference (src/hook.c), with its lines:
 *   - exported `dlsym` under GLIBC_2.2.5 and GLIBC_2.34, the real one obtained
 *     with dlvsym(RTLD_NEXT, ...)                                 :381-415,432-508,974-975
 *   - exported driver symbols cuInit, cuGetProcAddress{,_v2}, cuMemAlloc_v2,
 *     cuMemFree_v2, cuMemGetInfo_v2, cuLaunchKernel, cuMemcpy{,Async},
 *     cuMemcpy{HtoD,DtoH,DtoD}{,Async}_v2; the same set is what the hooked
 *     dlsym / cuGetProcAddress answer for                         :436-466,545-574
 *   - initialisation only from cuInit / cuGetProcAddress{,_v2}; every other
 *     hook returns CUDA_ERROR_NOT_INITIALIZED (3) before that     :539-540,654,756-757
 *   - cuMemGetInfo: free = total - 1536 MiB                       :698-746
 *   - cuMemAlloc: per-process cap = that "free"; over the cap ->
 *     CUDA_ERROR_OUT_OF_MEMORY (2) unless NVSHARE_ENABLE_SINGLE_OVERSUB
 *                                                                 :646-682
 *   - launches and memcpys wait for the GPU lock; launches run the adaptive
 *     cuCtxSynchronize window 1..2048 (x2 under 1 s, /2 from 1 s, reset from
 *     10 s)                                                       :766-840
 *   - driver errors are logged as "<fn> returned <name>: <string>" and returned
 *     unchanged                                                   :333-343
 *
 * What is different by design:
 *   - cuMemAlloc does NOT become cuMemAllocManaged.  It goes to the swap engine
 *     (engine.c): a VMM reservation whose 256 MiB chunks are mapped, copied out
 *     and unmapped explicitly around lock hand-offs.  The reference's path is
 *     still there as a mode (NVSHARE_ENGINE=uvm, and always when
 *     NVSHARE_ENABLE_SINGLE_OVERSUB is set, since a single process larger than
 *     HBM needs demand paging).
 *   - the interposed set is data: one table drives dlsym, cuGetProcAddress and
 *     the bootstrap, instead of three hand-written if-chains.
 *   - the gate also covers entry points a 2025 CUDA stack uses and the
 *     reference lets through ungated: cuLaunchKernelEx, cuLaunchCooperativeKernel,
 *     cuGraphLaunch, cuMemsetD*, cuMemcpy2D/3D/Peer -- with VMM memory an
 *     ungated touch of an evicted slab is a fatal fault, not a slow page-in.
 *   - cuGetProcAddress honours the per-thread-default-stream flag (each gated
 *     entry has a legacy and a per-thread forwarder) and answers
 *     "cuGetProcAddress" with the v2 hook when asked by a >= 12.0 runtime.
 *   - the allocation table is thread-safe (the reference's list is not).
 *   - the other ways of obtaining device memory are interposed too: cuMemAllocAsync,
 *     cuMemAllocFromPoolAsync, cuMemFreeAsync (stream-ordered) and cuMemAllocPitch.  The
 *     reference lets them through (src/hook.c:545-577 does not list them): memory obtained
 *     there is neither charged to the per-process cap nor swappable.  Here they take the
 *     same path as cuMemAlloc: cap check, then the swap engine (an allocation that is
 *     available at once is a valid stream-ordered allocation; a stream-ordered free first
 *     waits for the stream).
 *   - cuMemcpyHtoD/DtoH{,Async} on memory that is not on the GPU (swapped out or
 *     never materialised) do not wait for the lock: they are served from / into
 *     the pinned-host backing copy (host_io_bypass -> nvs_host_io, SURVEY 8f
 *     rank 3).  NVSHARE_LOCKFREE_COPY=0 gates them like the reference does.
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <dlfcn.h>
#include <inttypes.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "../../include/nvshare_engine.h"
#include "../../include/nvshare_wire.h"
#include "client.h"
#include "cuda_min.h"
#include "nvs_log.h"

#define EXPORT __attribute__((visibility("default")))

#define MEMINFO_RESERVE_BYTES (1536ull << 20) /* reference src/hook.c:45 */
#define SYNC_RESET_SECONDS 10                 /* reference src/hook.c:46 */
#define SYNC_STEPDOWN_SECONDS 1               /* reference src/hook.c:47 */
#define SYNC_WINDOW_MAX 2048                  /* reference src/hook.c:48 */
#define PTDS_FLAG 0x2ull /* CU_GET_PROC_ADDRESS_PER_THREAD_DEFAULT_STREAM */

/* ------------------------------------------------------------- state ---- */

static pthread_once_t once_lib = PTHREAD_ONCE_INIT;
static pthread_once_t once_client = PTHREAD_ONCE_INIT;
static void *cuda_lib;
static int single_oversub;
static int uvm_mode; /* reference mechanism instead of the swap engine */

static CUresult (*real_cuInit)(unsigned);
static CUresult (*real_cuGetProcAddress)(const char *, void **, int, cuuint64_t);
static CUresult (*real_cuGetProcAddress_v2)(const char *, void **, int, cuuint64_t,
					     CUdriverProcAddressQueryResult *);
static CUresult (*real_cuMemAllocManaged)(CUdeviceptr *, size_t, unsigned);
static CUresult (*real_cuMemAlloc)(CUdeviceptr *, size_t);
static CUresult (*real_cuMemFree)(CUdeviceptr);
static CUresult (*real_cuMemGetInfo)(size_t *, size_t *);
static CUresult (*real_cuGetErrorString)(CUresult, const char **);
static CUresult (*real_cuGetErrorName)(CUresult, const char **);
static CUresult (*real_cuCtxSetCurrent)(CUcontext);
static CUresult (*real_cuCtxGetCurrent)(CUcontext *);
static CUresult (*real_cuCtxSynchronize)(void);
static CUresult (*real_cuStreamIsCapturing)(CUstream, int *); /* optional */
static CUresult (*real_cuStreamSynchronize[2])(CUstream);      /* optional; [legacy, per-thread default stream] */
static CUresult (*real_cuMemFreeAsync[2])(CUdeviceptr, CUstream);

static pthread_mutex_t acct_mu = PTHREAD_MUTEX_INITIALIZER;
static size_t cap_bytes;     /* what cuMemGetInfo reports as free: the per-process cap */
static int cap_known;
static size_t sum_allocated; /* bytes the application currently holds via cuMemAlloc    */

static pthread_mutex_t window_mu = PTHREAD_MUTEX_INITIALIZER;
static int launches_since_sync;
static int sync_window = 1;

static pthread_mutex_t engine_mu = PTHREAD_MUTEX_INITIALIZER;
static nvs_engine *engine;
static CUcontext engine_ctx; /* the context the engine lives in: the first one an allocation was made from */
static int holds_lock;

/* ------------------------------------------------- the real dlsym ------- */

typedef void *(*dlsym_fn)(void *, const char *);

static void *real_dlsym_ver(int which, void *handle, const char *symbol)
{
	static const char *const versions[2] = {"GLIBC_2.2.5", "GLIBC_2.34"};
	static dlsym_fn cached[2];
	if (!cached[which]) {
		cached[which] = (dlsym_fn)dlvsym(RTLD_NEXT, "dlsym", versions[which]);
		if (!cached[which])
			nvs_fatal("cannot find the real dlsym@%s: %s", versions[which], dlerror());
	}
	return cached[which](handle, symbol);
}

static void *real_dlsym(void *handle, const char *symbol)
{
	static dlsym_fn f;
	if (!f) {
		f = (dlsym_fn)dlvsym(RTLD_NEXT, "dlsym", "GLIBC_2.2.5");
		if (!f)
			f = (dlsym_fn)dlvsym(RTLD_NEXT, "dlsym", "GLIBC_2.34");
		if (!f)
			nvs_fatal("cannot find the real dlsym: %s", dlerror());
	}
	return f(handle, symbol);
}

static void warn_if_error(CUresult r, const char *fn)
{
	if (r == CUDA_SUCCESS)
		return;
	const char *name = "?", *text = "?";
	if (real_cuGetErrorName)
		real_cuGetErrorName(r, &name);
	if (real_cuGetErrorString)
		real_cuGetErrorString(r, &text);
	nvs_warn("%s returned %s: %s", fn, name, text);
}

/* ------------------------------------------------- gated forwarders ----- */

/*
 * Each gated entry point gets two forwarders, [0] for the legacy default
 * stream and [1] for the per-thread default stream flavour the driver hands
 * out when cuGetProcAddress is called with PTDS_FLAG.  They differ only in
 * which real function they call.
 */
enum gate_id {
	G_cuLaunchKernel, G_cuLaunchKernelEx, G_cuLaunchCooperativeKernel, G_cuGraphLaunch,
	G_cuMemcpy, G_cuMemcpyAsync, G_cuMemcpyHtoD, G_cuMemcpyHtoDAsync, G_cuMemcpyDtoH,
	G_cuMemcpyDtoHAsync, G_cuMemcpyDtoD, G_cuMemcpyDtoDAsync,
	G_cuMemcpyPeer, G_cuMemcpyPeerAsync, G_cuMemcpy2D, G_cuMemcpy2DUnaligned, G_cuMemcpy2DAsync,
	G_cuMemcpy3D, G_cuMemcpy3DAsync, G_cuMemcpy3DPeer, G_cuMemcpy3DPeerAsync,
	G_cuMemsetD8, G_cuMemsetD16, G_cuMemsetD32, G_cuMemsetD8Async, G_cuMemsetD16Async, G_cuMemsetD32Async,
	G_cuMemsetD2D8, G_cuMemsetD2D16, G_cuMemsetD2D32, G_cuMemsetD2D8Async, G_cuMemsetD2D16Async,
	G_cuMemsetD2D32Async,
	G_COUNT
};
static void *gate_real[G_COUNT][2];

static void after_launch(CUstream s);

static int host_io_bypass(CUdeviceptr dev, const void *host, size_t n, int to_device, CUstream s);
static int touch_dst(CUdeviceptr dev, size_t n);
#define NO_BYPASS 0

/* `bypass`: an expression that is non-zero when the call has been served without
 * the GPU (nvs_host_io) and must therefore neither wait for the lock nor reach
 * the driver. */
#define GATED(name, is_launch, params, args) GATED_(name, is_launch, params, args, NO_BYPASS)
/* is_launch: 0, or LAUNCH_ON(stream expression) for entry points that submit kernels */
#define LAUNCH_ON(stream_expr) (1 + 0 * (uintptr_t)(launch_stream = (CUstream)(stream_expr)))
#define GATED_(name, is_launch, params, args, bypass)                                \
	static CUresult gate_##name##_impl(int flavour_, NVS_UNPAREN params)                \
	{                                                                            \
		typedef CUresult (*fn_t) params;                                     \
		fn_t real = (fn_t)gate_real[G_##name][flavour_];                            \
		if (!real)                                                           \
			real = (fn_t)gate_real[G_##name][0];                         \
		if (!real)                                                           \
			return CUDA_ERROR_NOT_INITIALIZED;                           \
		if (bypass)                                                          \
			return CUDA_SUCCESS;                                         \
		continue_with_lock();                                                \
		CUresult r = real args;                                              \
		warn_if_error(r, #name);                                             \
		CUstream launch_stream = NULL;                                       \
		if (is_launch)                                                       \
			after_launch(launch_stream);                                 \
		nvs_gate_leave();                                                    \
		return r;                                                            \
	}                                                                            \
	static CUresult gate_##name##_0 params { return gate_##name##_impl NVS_PREPEND(0, args); } \
	static CUresult gate_##name##_1 params { return gate_##name##_impl NVS_PREPEND(1, args); }

#define NVS_UNPAREN(...) __VA_ARGS__
#define NVS_PREPEND(x, ...) NVS_PREPEND_(x, NVS_UNPAREN __VA_ARGS__)
#define NVS_PREPEND_(x, ...) (x, __VA_ARGS__)

typedef unsigned int u32;
/* the leading fields of CUlaunchConfig (cuda.h): all this library needs is the stream */
struct nvs_launch_config_head {
	u32 grid[3], block[3], smem;
	CUstream stream;
};

GATED(cuLaunchKernel, LAUNCH_ON(s),
      (CUfunction f, u32 gx, u32 gy, u32 gz, u32 bx, u32 by, u32 bz, u32 smem, CUstream s, void **kp, void **extra),
      (f, gx, gy, gz, bx, by, bz, smem, s, kp, extra))
GATED(cuLaunchKernelEx, LAUNCH_ON(config ? ((const struct nvs_launch_config_head *)config)->stream : NULL),
      (const void *config, CUfunction f, void **kp, void **extra), (config, f, kp, extra))
GATED(cuLaunchCooperativeKernel, LAUNCH_ON(s),
      (CUfunction f, u32 gx, u32 gy, u32 gz, u32 bx, u32 by, u32 bz, u32 smem, CUstream s, void **kp),
      (f, gx, gy, gz, bx, by, bz, smem, s, kp))
GATED(cuGraphLaunch, LAUNCH_ON(s), (CUgraphExec g, CUstream s), (g, s))
GATED(cuMemcpy, 0, (CUdeviceptr dst, CUdeviceptr src, size_t n), (dst, src, n))
GATED(cuMemcpyAsync, 0, (CUdeviceptr dst, CUdeviceptr src, size_t n, CUstream s), (dst, src, n, s))
/* host<->device copies whose device side is swapped out are host<->host copies: no GPU, no lock */
GATED_(cuMemcpyHtoD, 0, (CUdeviceptr dst, const void *src, size_t n), (dst, src, n), host_io_bypass(dst, src, n, 1, NULL))
GATED_(cuMemcpyHtoDAsync, 0, (CUdeviceptr dst, const void *src, size_t n, CUstream s), (dst, src, n, s),
       host_io_bypass(dst, src, n, 1, s))
GATED_(cuMemcpyDtoH, 0, (void *dst, CUdeviceptr src, size_t n), (dst, src, n), host_io_bypass(src, dst, n, 0, NULL))
GATED_(cuMemcpyDtoHAsync, 0, (void *dst, CUdeviceptr src, size_t n, CUstream s), (dst, src, n, s),
       host_io_bypass(src, dst, n, 0, s))
GATED_(cuMemcpyDtoD, 0, (CUdeviceptr dst, CUdeviceptr src, size_t n), (dst, src, n), touch_dst(dst, n))
GATED_(cuMemcpyDtoDAsync, 0, (CUdeviceptr dst, CUdeviceptr src, size_t n, CUstream s), (dst, src, n, s), touch_dst(dst, n))
GATED(cuMemcpyPeer, 0, (CUdeviceptr dst, CUcontext dc, CUdeviceptr src, CUcontext sc, size_t n), (dst, dc, src, sc, n))
GATED(cuMemcpyPeerAsync, 0, (CUdeviceptr dst, CUcontext dc, CUdeviceptr src, CUcontext sc, size_t n, CUstream s),
      (dst, dc, src, sc, n, s))
GATED(cuMemcpy2D, 0, (const void *p), (p))
GATED(cuMemcpy2DUnaligned, 0, (const void *p), (p))
GATED(cuMemcpy2DAsync, 0, (const void *p, CUstream s), (p, s))
GATED(cuMemcpy3D, 0, (const void *p), (p))
GATED(cuMemcpy3DAsync, 0, (const void *p, CUstream s), (p, s))
GATED(cuMemcpy3DPeer, 0, (const void *p), (p))
GATED(cuMemcpy3DPeerAsync, 0, (const void *p, CUstream s), (p, s))
GATED_(cuMemsetD8, 0, (CUdeviceptr d, unsigned char v, size_t n), (d, v, n), touch_dst(d, n))
GATED_(cuMemsetD16, 0, (CUdeviceptr d, unsigned short v, size_t n), (d, v, n), touch_dst(d, 2 * n))
GATED_(cuMemsetD32, 0, (CUdeviceptr d, u32 v, size_t n), (d, v, n), touch_dst(d, 4 * n))
GATED_(cuMemsetD8Async, 0, (CUdeviceptr d, unsigned char v, size_t n, CUstream s), (d, v, n, s), touch_dst(d, n))
GATED_(cuMemsetD16Async, 0, (CUdeviceptr d, unsigned short v, size_t n, CUstream s), (d, v, n, s), touch_dst(d, 2 * n))
GATED_(cuMemsetD32Async, 0, (CUdeviceptr d, u32 v, size_t n, CUstream s), (d, v, n, s), touch_dst(d, 4 * n))
GATED(cuMemsetD2D8, 0, (CUdeviceptr d, size_t pitch, unsigned char v, size_t w, size_t h), (d, pitch, v, w, h))
GATED(cuMemsetD2D16, 0, (CUdeviceptr d, size_t pitch, unsigned short v, size_t w, size_t h), (d, pitch, v, w, h))
GATED(cuMemsetD2D32, 0, (CUdeviceptr d, size_t pitch, u32 v, size_t w, size_t h), (d, pitch, v, w, h))
GATED(cuMemsetD2D8Async, 0, (CUdeviceptr d, size_t pitch, unsigned char v, size_t w, size_t h, CUstream s),
      (d, pitch, v, w, h, s))
GATED(cuMemsetD2D16Async, 0, (CUdeviceptr d, size_t pitch, unsigned short v, size_t w, size_t h, CUstream s),
      (d, pitch, v, w, h, s))
GATED(cuMemsetD2D32Async, 0, (CUdeviceptr d, size_t pitch, u32 v, size_t w, size_t h, CUstream s),
      (d, pitch, v, w, h, s))

/* ------------------------------------------------- interposed table ----- */

EXPORT CUresult cuInit(unsigned flags);
EXPORT CUresult cuGetProcAddress(const char *symbol, void **pfn, int cudaVersion, cuuint64_t flags);
EXPORT CUresult cuGetProcAddress_v2(const char *symbol, void **pfn, int cudaVersion, cuuint64_t flags,
				    CUdriverProcAddressQueryResult *status);
EXPORT CUresult cuMemAlloc_v2(CUdeviceptr *dptr, size_t bytesize);
EXPORT CUresult cuMemFree_v2(CUdeviceptr dptr);
EXPORT CUresult cuMemGetInfo_v2(size_t *free_b, size_t *total_b);
EXPORT CUresult cuMemAllocPitch_v2(CUdeviceptr *dptr, size_t *pitch, size_t width_bytes, size_t height, unsigned elem);
EXPORT CUresult cuMemAllocAsync(CUdeviceptr *dptr, size_t bytesize, CUstream s);
EXPORT CUresult cuMemAllocFromPoolAsync(CUdeviceptr *dptr, size_t bytesize, void *pool, CUstream s);
EXPORT CUresult cuMemFreeAsync(CUdeviceptr dptr, CUstream s);
static CUresult hook_cuMemFreeAsync_ptsz(CUdeviceptr dptr, CUstream s);

struct entry {
	const char *base; /* name cuGetProcAddress is asked for          */
	const char *elf;  /* exported / dlsym name in libcuda            */
	void *hook[2];    /* [legacy, per-thread default stream]         */
	int gate;         /* index into gate_real, or -1                 */
	int reference;    /* 1: part of the reference's interposed set   */
	const char *ptds_suffix; /* "_ptsz", "_ptds" or NULL             */
};

#define E_GATE(name, elfname, ref, sfx) {#name, elfname, {(void *)gate_##name##_0, (void *)gate_##name##_1}, G_##name, ref, sfx}
#define E_PLAIN(name, elfname, fn) {#name, elfname, {(void *)fn, (void *)fn}, -1, 1, NULL}
#define E_PLAIN2(name, elfname, fn0, fn1) {#name, elfname, {(void *)fn0, (void *)fn1}, -1, 0, NULL}

static const struct entry ENTRIES[] = {
	E_PLAIN(cuInit, "cuInit", cuInit),
	E_PLAIN(cuGetProcAddress, "cuGetProcAddress", cuGetProcAddress),
	E_PLAIN(cuGetProcAddress_v2, "cuGetProcAddress_v2", cuGetProcAddress_v2),
	E_PLAIN(cuMemAlloc, "cuMemAlloc_v2", cuMemAlloc_v2),
	E_PLAIN(cuMemFree, "cuMemFree_v2", cuMemFree_v2),
	E_PLAIN(cuMemGetInfo, "cuMemGetInfo_v2", cuMemGetInfo_v2),
	E_GATE(cuLaunchKernel, "cuLaunchKernel", 1, "_ptsz"),
	E_GATE(cuMemcpy, "cuMemcpy", 1, "_ptds"),
	E_GATE(cuMemcpyAsync, "cuMemcpyAsync", 1, "_ptsz"),
	E_GATE(cuMemcpyHtoD, "cuMemcpyHtoD_v2", 1, "_ptds"),
	E_GATE(cuMemcpyHtoDAsync, "cuMemcpyHtoDAsync_v2", 1, "_ptsz"),
	E_GATE(cuMemcpyDtoH, "cuMemcpyDtoH_v2", 1, "_ptds"),
	E_GATE(cuMemcpyDtoHAsync, "cuMemcpyDtoHAsync_v2", 1, "_ptsz"),
	E_GATE(cuMemcpyDtoD, "cuMemcpyDtoD_v2", 1, "_ptds"),
	E_GATE(cuMemcpyDtoDAsync, "cuMemcpyDtoDAsync_v2", 1, "_ptsz"),
	/* beyond the reference's set (SURVEY 8f rank 2) */
	E_PLAIN2(cuMemAllocPitch, "cuMemAllocPitch_v2", cuMemAllocPitch_v2, cuMemAllocPitch_v2),
	E_PLAIN2(cuMemAllocAsync, "cuMemAllocAsync", cuMemAllocAsync, cuMemAllocAsync),
	E_PLAIN2(cuMemAllocFromPoolAsync, "cuMemAllocFromPoolAsync", cuMemAllocFromPoolAsync, cuMemAllocFromPoolAsync),
	E_PLAIN2(cuMemFreeAsync, "cuMemFreeAsync", cuMemFreeAsync, hook_cuMemFreeAsync_ptsz),
	E_GATE(cuLaunchKernelEx, "cuLaunchKernelEx", 0, "_ptsz"),
	E_GATE(cuLaunchCooperativeKernel, "cuLaunchCooperativeKernel", 0, "_ptsz"),
	E_GATE(cuGraphLaunch, "cuGraphLaunch", 0, "_ptsz"),
	E_GATE(cuMemcpyPeer, "cuMemcpyPeer", 0, "_ptds"),
	E_GATE(cuMemcpyPeerAsync, "cuMemcpyPeerAsync", 0, "_ptsz"),
	E_GATE(cuMemcpy2D, "cuMemcpy2D_v2", 0, "_ptds"),
	E_GATE(cuMemcpy2DUnaligned, "cuMemcpy2DUnaligned_v2", 0, "_ptds"),
	E_GATE(cuMemcpy2DAsync, "cuMemcpy2DAsync_v2", 0, "_ptsz"),
	E_GATE(cuMemcpy3D, "cuMemcpy3D_v2", 0, "_ptds"),
	E_GATE(cuMemcpy3DAsync, "cuMemcpy3DAsync_v2", 0, "_ptsz"),
	E_GATE(cuMemcpy3DPeer, "cuMemcpy3DPeer", 0, "_ptds"),
	E_GATE(cuMemcpy3DPeerAsync, "cuMemcpy3DPeerAsync", 0, "_ptsz"),
	E_GATE(cuMemsetD8, "cuMemsetD8_v2", 0, "_ptds"),
	E_GATE(cuMemsetD16, "cuMemsetD16_v2", 0, "_ptds"),
	E_GATE(cuMemsetD32, "cuMemsetD32_v2", 0, "_ptds"),
	E_GATE(cuMemsetD8Async, "cuMemsetD8Async", 0, "_ptsz"),
	E_GATE(cuMemsetD16Async, "cuMemsetD16Async", 0, "_ptsz"),
	E_GATE(cuMemsetD32Async, "cuMemsetD32Async", 0, "_ptsz"),
	E_GATE(cuMemsetD2D8, "cuMemsetD2D8_v2", 0, "_ptds"),
	E_GATE(cuMemsetD2D16, "cuMemsetD2D16_v2", 0, "_ptds"),
	E_GATE(cuMemsetD2D32, "cuMemsetD2D32_v2", 0, "_ptds"),
	E_GATE(cuMemsetD2D8Async, "cuMemsetD2D8Async", 0, "_ptsz"),
	E_GATE(cuMemsetD2D16Async, "cuMemsetD2D16Async", 0, "_ptsz"),
	E_GATE(cuMemsetD2D32Async, "cuMemsetD2D32Async", 0, "_ptsz"),
};
#define N_ENTRIES (sizeof(ENTRIES) / sizeof(ENTRIES[0]))

static const struct entry *find_by_elf(const char *name)
{
	for (size_t i = 0; i < N_ENTRIES; ++i)
		if (strcmp(ENTRIES[i].elf, name) == 0)
			return &ENTRIES[i];
	return NULL;
}

static const struct entry *find_by_base(const char *name)
{
	for (size_t i = 0; i < N_ENTRIES; ++i)
		if (strcmp(ENTRIES[i].base, name) == 0)
			return &ENTRIES[i];
	return NULL;
}

/* ------------------------------------------------------- bootstrap ------ */

static void *must_sym(const char *name)
{
	dlerror();
	void *p = real_dlsym(cuda_lib, name);
	const char *err = dlerror();
	if (err || !p)
		nvs_fatal("%s", err ? err : name);
	return p;
}

static void *engine_resolver(const char *symbol)
{
	return real_dlsym(cuda_lib, symbol);
}

static struct nvs_client_driver client_drv;

static void mark_exiting(void)
{
	__atomic_store_n(&nvs_process_exiting, 1, __ATOMIC_RELAXED);
}

static void bootstrap(void)
{
	if (getenv(NVS_ENV_DEBUG))
		nvs_debug_enabled = 1;
	atexit(mark_exiting);
	if (getenv("NVSHARE_ENABLE_SINGLE_OVERSUB")) {
		single_oversub = 1;
		uvm_mode = 1; /* a single process bigger than HBM needs demand paging */
		nvs_warn("Enabling GPU memory oversubscription for this application");
	}
	const char *mode = getenv("NVSHARE_ENGINE");
	if (mode && strcmp(mode, "uvm") == 0)
		uvm_mode = 1;

	void *nvml = dlopen("libnvidia-ml.so.1", RTLD_LAZY);
	if (nvml) {
		client_drv.nvmlInit = (nvmlReturn_t(*)(void))real_dlsym(nvml, "nvmlInit_v2");
		client_drv.nvmlDeviceGetHandleByIndex =
			(nvmlReturn_t(*)(unsigned, nvmlDevice_t *))real_dlsym(nvml, "nvmlDeviceGetHandleByIndex_v2");
		client_drv.nvmlDeviceGetUtilizationRates =
			(nvmlReturn_t(*)(nvmlDevice_t, nvmlUtilization_t *))real_dlsym(nvml, "nvmlDeviceGetUtilizationRates");
		client_drv.nvmlDeviceGetHandleByUUID =
			(nvmlReturn_t(*)(const char *, nvmlDevice_t *))real_dlsym(nvml, "nvmlDeviceGetHandleByUUID");
	}
	if (client_drv.nvmlInit && client_drv.nvmlDeviceGetHandleByIndex && client_drv.nvmlDeviceGetUtilizationRates) {
		nvs_debug("Found NVML");
	} else {
		client_drv.nvmlInit = NULL;
		nvs_debug("Could not find NVML");
	}

	cuda_lib = dlopen("libcuda.so.1", RTLD_LAZY);
	if (!cuda_lib)
		cuda_lib = dlopen("libcuda.so", RTLD_LAZY);
	if (!cuda_lib)
		nvs_fatal("%s", dlerror());

	real_cuInit = must_sym("cuInit");
	real_cuMemAllocManaged = must_sym("cuMemAllocManaged");
	real_cuMemAlloc = must_sym("cuMemAlloc_v2");
	real_cuMemFree = must_sym("cuMemFree_v2");
	real_cuMemGetInfo = must_sym("cuMemGetInfo_v2");
	real_cuGetErrorString = must_sym("cuGetErrorString");
	real_cuGetErrorName = must_sym("cuGetErrorName");
	real_cuCtxSetCurrent = must_sym("cuCtxSetCurrent");
	real_cuCtxGetCurrent = must_sym("cuCtxGetCurrent");
	real_cuCtxSynchronize = must_sym("cuCtxSynchronize");
	/* optional: runtimes < 11.3 / < 12.0 never ask for them */
	real_cuStreamIsCapturing = real_dlsym(cuda_lib, "cuStreamIsCapturing");
	real_cuStreamSynchronize[0] = real_dlsym(cuda_lib, "cuStreamSynchronize");
	real_cuStreamSynchronize[1] = real_dlsym(cuda_lib, "cuStreamSynchronize_ptsz");
	real_cuMemFreeAsync[0] = real_dlsym(cuda_lib, "cuMemFreeAsync");
	real_cuMemFreeAsync[1] = real_dlsym(cuda_lib, "cuMemFreeAsync_ptsz");
	real_cuGetProcAddress = real_dlsym(cuda_lib, "cuGetProcAddress");
	real_cuGetProcAddress_v2 = real_dlsym(cuda_lib, "cuGetProcAddress_v2");

	for (size_t i = 0; i < N_ENTRIES; ++i) {
		const struct entry *e = &ENTRIES[i];
		if (e->gate < 0)
			continue;
		/* the reference's set is mandatory (src/hook.c:224-268); the wider set is best effort */
		gate_real[e->gate][0] = e->reference ? must_sym(e->elf) : real_dlsym(cuda_lib, e->elf);
		if (e->ptds_suffix) {
			char name[96];
			snprintf(name, sizeof(name), "%s%s", e->elf, e->ptds_suffix);
			gate_real[e->gate][1] = real_dlsym(cuda_lib, name);
		}
	}
	dlerror();

	client_drv.cuInit = real_cuInit;
	client_drv.cuCtxGetCurrent = real_cuCtxGetCurrent;
	client_drv.cuCtxSetCurrent = real_cuCtxSetCurrent;
	client_drv.cuCtxSynchronize = real_cuCtxSynchronize;
	/* optional: which physical GPU the application is on (the idle detector's NVML query) */
	*(void **)&client_drv.cuCtxGetDevice = real_dlsym(cuda_lib, "cuCtxGetDevice");
	*(void **)&client_drv.cuDeviceGetUuid = real_dlsym(cuda_lib, "cuDeviceGetUuid_v2");
	if (!client_drv.cuDeviceGetUuid)
		*(void **)&client_drv.cuDeviceGetUuid = real_dlsym(cuda_lib, "cuDeviceGetUuid");
}

/* ----------------------------------------------- data path adapters ----- */

static int dp_fetch_all(void)
{
	if (NVS_EXITING())
		return 0;
	pthread_mutex_lock(&engine_mu);
	nvs_engine *e = engine;
	pthread_mutex_unlock(&engine_mu);
	if (!e)
		return 0;
	nvs_xfer_report rep;
	int rc = nvs_fetch_all(e, &rep);
	if (rc == NVS_E_SHUTDOWN || NVS_EXITING())
		return 0; /* the application is exiting: nothing left to keep consistent */
	if (rc != 0)
		nvs_warn("fetch failed: %s", nvs_strerror(rc));
	return rc;
}

static int dp_evict_impl(uint64_t min_bytes, int best_effort);
static int dp_evict(uint64_t min_bytes) { return dp_evict_impl(min_bytes, 0); }
static int dp_evict_best_effort(uint64_t min_bytes) { return dp_evict_impl(min_bytes, 1); }

static int dp_evict_impl(uint64_t min_bytes, int best_effort)
{
	if (NVS_EXITING())
		return 0;
	pthread_mutex_lock(&engine_mu);
	nvs_engine *e = engine;
	pthread_mutex_unlock(&engine_mu);
	if (!e)
		return 0;
	nvs_xfer_report rep;
	int rc = best_effort ? nvs_evict_best_effort(e, min_bytes, &rep) : nvs_evict(e, min_bytes, &rep);
	if (rc == NVS_E_SHUTDOWN || NVS_EXITING())
		return 0;
	if (rc != 0)
		nvs_warn("evict failed: %s", nvs_strerror(rc));
	return rc;
}

static void dp_evict_announce(void)
{
	if (NVS_EXITING())
		return;
	pthread_mutex_lock(&engine_mu);
	nvs_engine *e = engine;
	pthread_mutex_unlock(&engine_mu);
	if (e)
		nvs_evict_announce(e);
}

static uint64_t dp_nonresident_mib(void)
{
	pthread_mutex_lock(&engine_mu);
	nvs_engine *e = engine;
	pthread_mutex_unlock(&engine_mu);
	nvs_stats st;
	if (!e || nvs_get_stats(e, &st) != 0)
		return 0;
	return (st.swapped_bytes + st.unbacked_bytes) >> 20;
}

static uint64_t dp_free_hbm_mib(void)
{
	size_t free_b = 0, total_b = 0;
	if (!real_cuMemGetInfo || real_cuMemGetInfo(&free_b, &total_b) != CUDA_SUCCESS)
		return 0;
	return (uint64_t)free_b >> 20;
}

static uint64_t dp_total_hbm_mib(void)
{
	size_t free_b = 0, total_b = 0;
	if (!real_cuMemGetInfo || real_cuMemGetInfo(&free_b, &total_b) != CUDA_SUCCESS)
		return 0;
	return (uint64_t)total_b >> 20;
}

static void on_engine_pressure(void *user, uint64_t bytes)
{
	(void)user;
	nvs_client_pressure((bytes + (1u << 20) - 1) >> 20);
}

static void dp_lock_state(int v)
{
	pthread_mutex_lock(&engine_mu);
	__atomic_store_n(&holds_lock, v, __ATOMIC_RELAXED); /* host_io_bypass() reads it without the mutex */
	if (engine)
		nvs_set_resident_mode(engine, v);
	pthread_mutex_unlock(&engine_mu);
}

static void reset_sync_window(void)
{
	pthread_mutex_lock(&window_mu);
	sync_window = 1;
	pthread_mutex_unlock(&window_mu);
}

static void start_client(void)
{
	static const struct nvs_client_datapath dp = {dp_fetch_all, dp_evict, dp_nonresident_mib, dp_lock_state,
						       dp_free_hbm_mib, dp_total_hbm_mib, dp_evict_best_effort, dp_evict_announce};
	nvs_client_on_context_sync = reset_sync_window;
	nvs_client_start(&client_drv, uvm_mode ? NULL : &dp);
}

static void ensure_init(void)
{
	nvs_must(pthread_once(&once_lib, bootstrap) == 0);
	nvs_must(pthread_once(&once_client, start_client) == 0);
}

/* The engine binds to the application's context, so it can only be created
 * once the application has one (its first cuMemAlloc).  NULL: no context yet. */
static nvs_engine *engine_get(void)
{
	pthread_mutex_lock(&engine_mu);
	if (!engine && !uvm_mode) {
		CUcontext ctx = NULL;
		if (real_cuCtxGetCurrent(&ctx) == CUDA_SUCCESS && ctx != NULL) {
			nvs_engine_config cfg;
			nvs_engine_default_config(&cfg);
			cfg.resolve = engine_resolver;
			cfg.pressure_cb = on_engine_pressure;
			/* one pinned-host backing store for all clients of this scheduler */
			static char pool_path[256];
			const char *pool = getenv("NVSHARE_POOL");
			if (!(pool && strcmp(pool, "private") == 0) && nvs_pool_path(pool_path, sizeof(pool_path)) == 0)
				cfg.shared_pool_path = pool_path;
			nvs_engine *made = NULL; /* published below: lock-free readers (lent_now, the copy bypass) load `engine` atomically */
			int rc = nvs_engine_create(&cfg, &made);
			if (rc == NVS_E_NO_KERNEL || rc == NVS_E_NO_DRIVER) {
				/* not an H100 (only the sm_90a image is embedded), or a driver without the VMM entry
				 * points: the drop-in still has to work, so this process runs on the reference's
				 * managed-memory mechanism (cuMemAllocManaged + UVM faults) like NVSHARE_ENGINE=uvm */
				nvs_warn("swap engine unavailable on this GPU/driver (%s): falling back to the reference's "
					 "managed-memory mechanism for this process", nvs_strerror(rc));
				uvm_mode = 1;
			} else if (rc != 0) {
				nvs_fatal("swap engine could not start (%s); set NVSHARE_ENGINE=uvm to run with "
					  "the reference's managed-memory mechanism instead", nvs_strerror(rc));
			} else {
				nvs_set_resident_mode(made, holds_lock);
				engine_ctx = ctx;
				__atomic_store_n(&engine, made, __ATOMIC_RELEASE);
			}
		}
	}
	nvs_engine *e = engine;
	pthread_mutex_unlock(&engine_mu);
	return e;
}

/*
 * SURVEY 8f rank 3.  A client that does not hold the GPU lock has nothing on the
 * GPU that could race with this: its context was drained before its memory was
 * swapped out, and everything it submits is parked at the gate.  So a copy
 * between host memory and a swapped-out (or never materialised) device range is
 * served by the engine from / into the pinned-host backing copy, and a client
 * loading its inputs no longer takes the GPU away from the one computing.
 * The engine re-checks the state of the range under its own lock: if LOCK_OK got
 * there first the range is resident and the call goes down the gated path.
 * NVSHARE_LOCKFREE_COPY=0 turns it off.
 */
/* Recency hint for partial evictions: the application is writing this range from the host side of
 * the API.  Always 0: the call itself still goes through the gate. */
static int touch_dst(CUdeviceptr dev, size_t n)
{
	nvs_engine *e = __atomic_load_n(&engine, __ATOMIC_ACQUIRE);
	if (e && n)
		nvs_touch(e, (uint64_t)dev, (uint64_t)n);
	return 0;
}

static int host_io_bypass(CUdeviceptr dev, const void *host, size_t n, int to_device, CUstream s)
{
	static int enabled = -1;
	if (to_device)
		touch_dst(dev, n);
	if (enabled < 0) {
		const char *v = getenv("NVSHARE_LOCKFREE_COPY");
		enabled = !(v && *v && atoi(v) == 0);
	}
	if (!enabled || n == 0 || !host || __atomic_load_n(&holds_lock, __ATOMIC_RELAXED))
		return 0;
	nvs_engine *e = __atomic_load_n(&engine, __ATOMIC_ACQUIRE);
	if (!e)
		return 0;
	if (s && real_cuStreamIsCapturing) {
		/* a copy issued into a capturing stream is a graph node to be recorded, not work to do now */
		int capturing = 0;
		if (real_cuStreamIsCapturing(s, &capturing) != CUDA_SUCCESS || capturing != 0)
			return 0;
	}
	int rc = nvs_host_io(e, (uint64_t)dev, (void *)(uintptr_t)host, (uint64_t)n, to_device);
	if (rc == 0)
		nvs_debug("%s of %zu bytes served from the backing copy, no lock needed", to_device ? "HtoD" : "DtoH", n);
	return rc == 0;
}

/* ------------------------------------------------- launch window -------- */

/* Reference src/hook.c:782-838: keep the amount of queued GPU work bounded so a
 * DROP_LOCK can be honoured quickly. */
static void after_launch(CUstream s)
{
	/* A launch into a capturing stream records a graph node, it queues no work -- and a
	 * cuCtxSynchronize here would be an illegal call that invalidates the capture
	 * (torch.cuda.graphs, cuBLAS graph capture).  The reference synchronises regardless
	 * (src/hook.c:808): stream capture under it fails. */
	if (s && real_cuStreamIsCapturing) {
		int capturing = 0;
		if (real_cuStreamIsCapturing(s, &capturing) == CUDA_SUCCESS && capturing != 0)
			return;
	}
	pthread_mutex_lock(&window_mu);
	if (++launches_since_sync >= sync_window) {
		struct timespec a, b;
		clock_gettime(CLOCK_MONOTONIC, &a);
		CUresult r = real_cuCtxSynchronize();
		warn_if_error(r, "cuCtxSynchronize");
		clock_gettime(CLOCK_MONOTONIC, &b);
		long secs = b.tv_sec - a.tv_sec - (b.tv_nsec < a.tv_nsec ? 1 : 0);
		if (secs >= SYNC_RESET_SECONDS)
			sync_window = 1;
		else if (secs >= SYNC_STEPDOWN_SECONDS)
			sync_window = sync_window / 2 > 1 ? sync_window / 2 : 1;
		else
			sync_window = sync_window * 2 < SYNC_WINDOW_MAX ? sync_window * 2 : SYNC_WINDOW_MAX;
		nvs_debug("Pending Kernel Window is %d.", sync_window);
		launches_since_sync = 0;
	}
	pthread_mutex_unlock(&window_mu);
}

/* ------------------------------------------- UVM-mode allocation list --- */

struct uvm_alloc {
	CUdeviceptr ptr;
	size_t size;
	struct uvm_alloc *next;
};
static struct uvm_alloc *uvm_buckets[256];

static inline unsigned uvm_hash(CUdeviceptr p)
{
	return (unsigned)((p >> 9) * 2654435761u) >> 24;
}

static void uvm_insert(CUdeviceptr p, size_t n)
{
	struct uvm_alloc *a = malloc(sizeof(*a));
	nvs_must(a != NULL);
	a->ptr = p;
	a->size = n;
	unsigned h = uvm_hash(p);
	a->next = uvm_buckets[h];
	uvm_buckets[h] = a;
}

static size_t uvm_remove(CUdeviceptr p)
{
	unsigned h = uvm_hash(p);
	for (struct uvm_alloc **pp = &uvm_buckets[h]; *pp; pp = &(*pp)->next)
		if ((*pp)->ptr == p) {
			struct uvm_alloc *a = *pp;
			size_t n = a->size;
			*pp = a->next;
			free(a);
			return n;
		}
	return 0;
}

/* ------------------------------------------------- exported hooks ------- */

CUresult cuInit(unsigned flags)
{
	ensure_init();
	CUresult r = real_cuInit(flags);
	warn_if_error(r, "cuInit");
	return r;
}

/* HBM of the GPU this process computes on that clients of OTHER GPUs use as backing right now (the
 * peer tier of their engines; gpu_ledger.h).  The reference knows one GPU and one kind of tenant
 * (src/hook.c:662); here what a GPU has lent is not there for its own clients, so it comes off what
 * they are told is free and off their cap.  0 until this process has an engine, and whenever nobody
 * lends -- the reference's numbers exactly. */
static size_t lent_now(void)
{
	nvs_engine *e = __atomic_load_n(&engine, __ATOMIC_ACQUIRE);
	return e ? (size_t)nvs_gpu_lent_bytes(e) : 0;
}

static CUresult meminfo(size_t *free_b, size_t *total_b, size_t lent)
{
	if (!real_cuMemGetInfo)
		return CUDA_ERROR_NOT_INITIALIZED;
	CUresult r = real_cuMemGetInfo(free_b, total_b);
	warn_if_error(r, "cuMemGetInfo_v2");
	nvs_debug("real_cuMemGetInfo returned free=%.2f MiB, total=%.2f MiB", *free_b / 1048576.0,
		  *total_b / 1048576.0);
	/* hide a fixed slice for contexts and libraries, whatever is really free */
	*free_b = *total_b - (size_t)MEMINFO_RESERVE_BYTES;
	*free_b = *free_b > lent ? *free_b - lent : 0;
	nvs_debug("nvshare's cuMemGetInfo returning free=%.2f MiB, total=%.2f MiB", *free_b / 1048576.0,
		  *total_b / 1048576.0);
	return r;
}

CUresult cuMemGetInfo_v2(size_t *free_b, size_t *total_b)
{
	return meminfo(free_b, total_b, lent_now());
}

CUresult cuMemAlloc_v2(CUdeviceptr *dptr, size_t bytesize)
{
	if (!real_cuMemAllocManaged)
		return CUDA_ERROR_NOT_INITIALIZED;
	pthread_mutex_lock(&acct_mu);
	if (!cap_known) {
		size_t total = 0;
		CUresult r = meminfo(&cap_bytes, &total, 0); /* the fixed part; what the GPU has lent is looked up per request */
		warn_if_error(r, "cuMemGetInfo_v2");
		cap_known = 1;
	}
	/* (the reference's `sum_allocated + bytesize > cap`, src/hook.c:662, without the wrap-around of a huge request) */
	const size_t lent = lent_now();
	const size_t cap_now = cap_bytes > lent ? cap_bytes - lent : 0;
	if (sum_allocated > cap_now || bytesize > cap_now - sum_allocated) {
		if (!single_oversub) {
			pthread_mutex_unlock(&acct_mu);
			return CUDA_ERROR_OUT_OF_MEMORY;
		}
		nvs_warn("Memory allocations exceeded physical GPU memory capacity. This can cause extreme"
			 " performance degradation!");
	}
	sum_allocated += bytesize; /* reserved at the check: two threads cannot both pass it on the same room */
	pthread_mutex_unlock(&acct_mu);

	nvs_debug("cuMemAlloc requested %zu bytes", bytesize);
	CUresult r;
	nvs_engine *e = uvm_mode ? NULL : engine_get(); /* may switch uvm_mode on (no usable engine here) */
	int foreign = 0;
	if (e) {
		/* One engine, one context, one GPU -- the reference's "single context / single device" (its
		 * README) with the difference that managed memory does not care which context asks for it and
		 * ours does: an allocation made from ANOTHER context (a second GPU in the same process) must
		 * not come out of the first GPU's engine.  It gets what the reference would have given it. */
		CUcontext cur = NULL;
		if (real_cuCtxGetCurrent(&cur) == CUDA_SUCCESS && cur != NULL && cur != engine_ctx) {
			static int warned;
			if (!__atomic_exchange_n(&warned, 1, __ATOMIC_RELAXED))
				nvs_warn("allocation from a second CUDA context: only the first context's memory is swapped explicitly, "
					 "this one is managed memory like under the reference");
			foreign = 1;
		}
	}
	if (uvm_mode || foreign) {
		e = NULL;
		r = real_cuMemAllocManaged(dptr, bytesize, CU_MEM_ATTACH_GLOBAL);
		warn_if_error(r, "cuMemAllocManaged");
	} else if (e) {
		uint64_t p = 0;
		int rc = nvs_alloc(e, &p, bytesize);
		r = rc >= 0 ? (CUresult)rc : CUDA_ERROR_UNKNOWN;
		if (r == CUDA_SUCCESS)
			*dptr = p;
		else
			nvs_warn("cuMemAlloc_v2 (swap engine) returned %d: %s", (int)r, nvs_strerror(rc));
	} else {
		/* no current context: let the driver produce its own error */
		r = real_cuMemAlloc(dptr, bytesize);
		warn_if_error(r, "cuMemAlloc_v2");
		if (r == CUDA_SUCCESS)
			nvs_warn("allocation made without a current context is not swappable");
	}
	pthread_mutex_lock(&acct_mu);
	if (r == CUDA_SUCCESS) {
		if (uvm_mode || !e)
			uvm_insert(*dptr, bytesize);
		nvs_debug("Total allocated memory on GPU is %.2f MiB", sum_allocated / 1048576.0);
	} else {
		sum_allocated -= bytesize;
	}
	pthread_mutex_unlock(&acct_mu);
	return r;
}

CUresult cuMemFree_v2(CUdeviceptr dptr)
{
	if (!real_cuMemFree)
		return CUDA_ERROR_NOT_INITIALIZED;
	pthread_mutex_lock(&engine_mu);
	nvs_engine *e = engine;
	pthread_mutex_unlock(&engine_mu);
	if (e) {
		uint64_t bytes = 0;
		int rc = nvs_free_sized(e, dptr, &bytes);
		if (rc == 0) {
			pthread_mutex_lock(&acct_mu);
			sum_allocated -= bytes;
			nvs_debug("Total allocated memory on GPU is %.2f MiB", sum_allocated / 1048576.0);
			pthread_mutex_unlock(&acct_mu);
			return CUDA_SUCCESS;
		}
		if (rc != NVS_E_NOT_OURS)
			return rc > 0 ? (CUresult)rc : CUDA_ERROR_UNKNOWN;
	}
	CUresult r = real_cuMemFree(dptr);
	if (r == CUDA_SUCCESS) {
		pthread_mutex_lock(&acct_mu);
		sum_allocated -= uvm_remove(dptr);
		pthread_mutex_unlock(&acct_mu);
	}
	return r;
}

/* ---- the other allocation entry points (SURVEY 8f rank 2; not in the reference's set) ---- */

CUresult cuMemAllocPitch_v2(CUdeviceptr *dptr, size_t *pitch, size_t width_bytes, size_t height, unsigned elem)
{
	if (!real_cuMemAllocManaged)
		return CUDA_ERROR_NOT_INITIALIZED;
	if (!dptr || !pitch || width_bytes == 0 || height == 0 || !(elem == 4 || elem == 8 || elem == 16))
		return CUDA_ERROR_INVALID_VALUE;
	/* what the driver does on every GPU that has VMM: rows padded to 512 bytes */
	if (width_bytes > SIZE_MAX - 511)
		return CUDA_ERROR_OUT_OF_MEMORY;
	const size_t p = (width_bytes + 511) & ~(size_t)511;
	if (p > SIZE_MAX / height) /* (a product that wraps must not come back as a small allocation) */
		return CUDA_ERROR_OUT_OF_MEMORY;
	CUresult r = cuMemAlloc_v2(dptr, p * height);
	if (r == CUDA_SUCCESS)
		*pitch = p;
	return r;
}

/* Stream-ordered allocation: "available when the stream gets there".  Memory that is available
 * at once satisfies that, so these are cuMemAlloc with the cap check and the swap engine behind
 * it; the memory pool argument only says where the driver would have taken the memory from. */
CUresult cuMemAllocAsync(CUdeviceptr *dptr, size_t bytesize, CUstream s)
{
	(void)s;
	return cuMemAlloc_v2(dptr, bytesize);
}

CUresult cuMemAllocFromPoolAsync(CUdeviceptr *dptr, size_t bytesize, void *pool, CUstream s)
{
	(void)pool;
	(void)s;
	return cuMemAlloc_v2(dptr, bytesize);
}

/* Stream-ordered free: everything queued on the stream before the call may still use the memory.
 * Ours is released on the host side, so the stream is drained first (the driver's own free of
 * memory we did not hand out keeps its asynchronous semantics). */
static CUresult free_async(int flavour, CUdeviceptr dptr, CUstream s)
{
	if (!real_cuMemFree)
		return CUDA_ERROR_NOT_INITIALIZED;
	nvs_engine *e = __atomic_load_n(&engine, __ATOMIC_ACQUIRE);
	int ours = 0;
	pthread_mutex_lock(&acct_mu);
	for (struct uvm_alloc *a = uvm_buckets[uvm_hash(dptr)]; a && !ours; a = a->next)
		ours = a->ptr == dptr;
	pthread_mutex_unlock(&acct_mu);
	if (!ours && e && nvs_lookup(e, (uint64_t)dptr, NULL) == 0)
		ours = 1;
	if (!ours) {
		if (real_cuMemFreeAsync[flavour] || real_cuMemFreeAsync[0])
			return (real_cuMemFreeAsync[flavour] ? real_cuMemFreeAsync[flavour] : real_cuMemFreeAsync[0])(dptr, s);
		return CUDA_ERROR_INVALID_VALUE;
	}
	if (s && real_cuStreamIsCapturing) {
		/* Inside a capture the driver would record a free NODE; memory of ours cannot be released by a
		 * graph, and synchronising the stream would invalidate the capture.  Refuse, loudly, and leave
		 * the capture intact: the memory stays allocated until cuMemFree. */
		int capturing = 0;
		if (real_cuStreamIsCapturing(s, &capturing) == CUDA_SUCCESS && capturing != 0) {
			nvs_warn("cuMemFreeAsync inside a stream capture is not supported for swappable memory; free it outside the capture");
			return CUDA_ERROR_NOT_SUPPORTED;
		}
	}
	CUresult (*sync)(CUstream) = real_cuStreamSynchronize[flavour] ? real_cuStreamSynchronize[flavour] : real_cuStreamSynchronize[0];
	CUresult r = sync ? sync(s) : real_cuCtxSynchronize();
	if (r != CUDA_SUCCESS)
		return r;
	return cuMemFree_v2(dptr);
}

CUresult cuMemFreeAsync(CUdeviceptr dptr, CUstream s) { return free_async(0, dptr, s); }
static CUresult hook_cuMemFreeAsync_ptsz(CUdeviceptr dptr, CUstream s) { return free_async(1, dptr, s); }

/* reference-exported names of the gated set: the legacy-stream forwarders */
EXPORT CUresult cuLaunchKernel(CUfunction f, u32 gx, u32 gy, u32 gz, u32 bx, u32 by, u32 bz, u32 smem, CUstream s,
			       void **kp, void **extra)
{
	return gate_cuLaunchKernel_0(f, gx, gy, gz, bx, by, bz, smem, s, kp, extra);
}
EXPORT CUresult cuMemcpy(CUdeviceptr dst, CUdeviceptr src, size_t n) { return gate_cuMemcpy_0(dst, src, n); }
EXPORT CUresult cuMemcpyAsync(CUdeviceptr dst, CUdeviceptr src, size_t n, CUstream s) { return gate_cuMemcpyAsync_0(dst, src, n, s); }
EXPORT CUresult cuMemcpyHtoD_v2(CUdeviceptr dst, const void *src, size_t n) { return gate_cuMemcpyHtoD_0(dst, src, n); }
EXPORT CUresult cuMemcpyHtoDAsync_v2(CUdeviceptr dst, const void *src, size_t n, CUstream s) { return gate_cuMemcpyHtoDAsync_0(dst, src, n, s); }
EXPORT CUresult cuMemcpyDtoH_v2(void *dst, CUdeviceptr src, size_t n) { return gate_cuMemcpyDtoH_0(dst, src, n); }
EXPORT CUresult cuMemcpyDtoHAsync_v2(void *dst, CUdeviceptr src, size_t n, CUstream s) { return gate_cuMemcpyDtoHAsync_0(dst, src, n, s); }
EXPORT CUresult cuMemcpyDtoD_v2(CUdeviceptr dst, CUdeviceptr src, size_t n) { return gate_cuMemcpyDtoD_0(dst, src, n); }
EXPORT CUresult cuMemcpyDtoDAsync_v2(CUdeviceptr dst, CUdeviceptr src, size_t n, CUstream s) { return gate_cuMemcpyDtoDAsync_0(dst, src, n, s); }
/* wider set, exported for pure driver-API applications */
EXPORT CUresult cuLaunchKernelEx(const void *c, CUfunction f, void **kp, void **extra) { return gate_cuLaunchKernelEx_0(c, f, kp, extra); }
EXPORT CUresult cuLaunchCooperativeKernel(CUfunction f, u32 gx, u32 gy, u32 gz, u32 bx, u32 by, u32 bz, u32 smem,
					  CUstream s, void **kp)
{
	return gate_cuLaunchCooperativeKernel_0(f, gx, gy, gz, bx, by, bz, smem, s, kp);
}
EXPORT CUresult cuGraphLaunch(CUgraphExec g, CUstream s) { return gate_cuGraphLaunch_0(g, s); }
EXPORT CUresult cuMemsetD8_v2(CUdeviceptr d, unsigned char v, size_t n) { return gate_cuMemsetD8_0(d, v, n); }
EXPORT CUresult cuMemsetD16_v2(CUdeviceptr d, unsigned short v, size_t n) { return gate_cuMemsetD16_0(d, v, n); }
EXPORT CUresult cuMemsetD32_v2(CUdeviceptr d, u32 v, size_t n) { return gate_cuMemsetD32_0(d, v, n); }
EXPORT CUresult cuMemsetD8Async(CUdeviceptr d, unsigned char v, size_t n, CUstream s) { return gate_cuMemsetD8Async_0(d, v, n, s); }
EXPORT CUresult cuMemsetD16Async(CUdeviceptr d, unsigned short v, size_t n, CUstream s) { return gate_cuMemsetD16Async_0(d, v, n, s); }
EXPORT CUresult cuMemsetD32Async(CUdeviceptr d, u32 v, size_t n, CUstream s) { return gate_cuMemsetD32Async_0(d, v, n, s); }

/* ------------------------------------------------- symbol lookup -------- */

CUresult cuGetProcAddress_v2(const char *symbol, void **pfn, int cudaVersion, cuuint64_t flags,
			     CUdriverProcAddressQueryResult *status)
{
	ensure_init();
	if (!real_cuGetProcAddress_v2)
		return CUDA_ERROR_NOT_INITIALIZED;
	const struct entry *e = find_by_base(symbol);
	if (!e)
		return real_cuGetProcAddress_v2(symbol, pfn, cudaVersion, flags, status);
	const int v = (flags & PTDS_FLAG) ? 1 : 0;
	if (e->gate >= 0 && !gate_real[e->gate][v]) {
		/* learn the real function for this flavour from the driver itself */
		void *p = NULL;
		CUdriverProcAddressQueryResult st = CU_GET_PROC_ADDRESS_SUCCESS;
		CUresult r = real_cuGetProcAddress_v2(symbol, &p, cudaVersion, flags, &st);
		if (r != CUDA_SUCCESS || !p) { /* this driver does not have it: say so */
			*pfn = p;
			if (status)
				*status = st;
			return r;
		}
		gate_real[e->gate][v] = p;
	}
	if (e->hook[0] == (void *)cuGetProcAddress && cudaVersion >= 12000)
		*pfn = (void *)cuGetProcAddress_v2; /* what a 12.x runtime means by "cuGetProcAddress" */
	else
		*pfn = e->hook[v];
	if (status)
		*status = CU_GET_PROC_ADDRESS_SUCCESS;
	return CUDA_SUCCESS;
}

CUresult cuGetProcAddress(const char *symbol, void **pfn, int cudaVersion, cuuint64_t flags)
{
	ensure_init();
	if (!real_cuGetProcAddress)
		return CUDA_ERROR_NOT_INITIALIZED;
	const struct entry *e = find_by_base(symbol);
	if (!e)
		return real_cuGetProcAddress(symbol, pfn, cudaVersion, flags);
	const int v = (flags & PTDS_FLAG) ? 1 : 0;
	if (e->gate >= 0 && !gate_real[e->gate][v]) {
		void *p = NULL;
		CUresult r = real_cuGetProcAddress(symbol, &p, cudaVersion, flags);
		if (r != CUDA_SUCCESS || !p) {
			*pfn = p;
			return r;
		}
		gate_real[e->gate][v] = p;
	}
	*pfn = e->hook[v];
	return CUDA_SUCCESS;
}

static void *hooked_dlsym(int version, void *handle, const char *symbol)
{
	if (symbol && symbol[0] == 'c' && symbol[1] == 'u') {
		const struct entry *e = find_by_elf(symbol);
		if (e)
			return e->hook[0];
	}
	return real_dlsym_ver(version, handle, symbol);
}

EXPORT void *nvs_dlsym_225(void *handle, const char *symbol)
{
	return hooked_dlsym(0, handle, symbol);
}

EXPORT void *nvs_dlsym_234(void *handle, const char *symbol)
{
	return hooked_dlsym(1, handle, symbol);
}

#ifndef NVS_NO_DLSYM_EXPORT /* ThreadSanitizer builds (tools/sanitize.sh tsan): its start-up cannot live with an interposed dlsym */
__asm__(".symver nvs_dlsym_225, dlsym@@GLIBC_2.2.5");
__asm__(".symver nvs_dlsym_234, dlsym@GLIBC_2.34");
#endif
