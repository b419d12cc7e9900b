/*
 * fake_cuda.c -- TEST DOUBLE for libcuda.so.1 (built as oracle/_ref/fakecuda/
 * libcuda.so.1).  TEST INFRASTRUCTURE ONLY: nothing in the product links or
 * loads this; the CPU test-suite puts its directory on LD_LIBRARY_PATH so that
 * the reference's libnvshare.so AND ours can be exercised without a GPU.
 *
 * What it emulates, and how faithfully:
 *   - "HBM" is host memory with a capacity (FAKE_CUDA_TOTAL_MIB, default 4096).
 *     Physical use is accounted in a ledger that can be shared between
 *     processes (FAKE_CUDA_LEDGER=<file>), so that "client B cannot map until
 *     client A has released" is testable on CPU.
 *   - the VMM API is emulated with mmap: cuMemAddressReserve -> PROT_NONE
 *     reservation, cuMemCreate -> memfd, cuMemMap -> MAP_FIXED mapping of the
 *     memfd, cuMemUnmap -> back to PROT_NONE.  Touching an evicted slab
 *     therefore SEGFAULTS, like a real GPU raising an Xid on an unmapped VA:
 *     a missing fetch cannot pass a test silently.
 *   - cuLaunchKernel understands the four entry points of
 *     nvshare_b200/csrc/slab_copy.cu (by name) and executes their byte
 *     semantics with memcpy / the same SplitMix64 pattern; any other
 *     CUfunction is only counted.  Streams run synchronously.
 *   - every call is appended to FAKE_CUDA_TRACE (one line each) so that the
 *     driver-call trace of the reference and of our library can be compared.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <errno.h>
#include <fcntl.h>
#include <pthread.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>
#include <sys/mman.h>
#include <sys/resource.h>
#include <sys/stat.h>

typedef int CUresult;
typedef unsigned long long CUdeviceptr;
typedef int CUdevice;
typedef void *CUcontext, *CUstream, *CUfunction, *CUmodule, *CUevent;
typedef unsigned long long CUmemGenericAllocationHandle;

#define OK 0
#define E_INVALID 1
#define E_OOM 2
#define E_NOT_INIT 3
#define E_NOT_FOUND 500

#define SLAB (2ull << 20)

#include "slab_hash_ref.h"

#define FAKE_MAX_GPUS 16
struct ledger {
	/* physical "HBM" bytes in use across all attached processes, per physical GPU.  [0] is the GPU
	 * every single-GPU test runs on; the others only exist for the peer-tier tests. */
	volatile uint64_t used[FAKE_MAX_GPUS];
};

static pthread_mutex_t g_mu = PTHREAD_MUTEX_INITIALIZER;
static struct ledger g_private_ledger, *g_ledger = &g_private_ledger;
static uint64_t g_total;
/* FAKE_CUDA_VISIBLE="2,0,1": ordinal -> physical GPU, like CUDA_VISIBLE_DEVICES (default: identity);
 * FAKE_CUDA_DEVICE=<ordinal>: the GPU the (one) context of this process is on (default 0) */
static int g_phys_of[FAKE_MAX_GPUS];
static int g_cur_ordinal;
static int phys_of(int ordinal) { return ordinal >= 0 && ordinal < FAKE_MAX_GPUS ? g_phys_of[ordinal] : 0; }
static int g_inited;
static FILE *g_trace;
static int g_ctx_token;
static __thread void *t_ctx_stack[16];
static __thread int t_ctx_depth;

static void setup_once(void)
{
	static int done;
	if (done)
		return;
	done = 1;
	/* one memfd per mapped chunk: lift the descriptor limit as far as allowed */
	struct rlimit rl;
	if (getrlimit(RLIMIT_NOFILE, &rl) == 0 && rl.rlim_cur < rl.rlim_max) {
		rl.rlim_cur = rl.rlim_max;
		setrlimit(RLIMIT_NOFILE, &rl);
	}
	const char *t = getenv("FAKE_CUDA_TOTAL_MIB");
	g_total = (t ? strtoull(t, NULL, 0) : 4096ull) << 20;
	for (int i = 0; i < FAKE_MAX_GPUS; ++i)
		g_phys_of[i] = i;
	const char *vis = getenv("FAKE_CUDA_VISIBLE");
	if (vis && *vis) {
		char buf[128], *save = NULL;
		snprintf(buf, sizeof(buf), "%s", vis);
		int k = 0;
		for (char *tok = strtok_r(buf, ",", &save); tok && k < FAKE_MAX_GPUS; tok = strtok_r(NULL, ",", &save))
			g_phys_of[k++] = atoi(tok) & (FAKE_MAX_GPUS - 1);
	}
	const char *cur = getenv("FAKE_CUDA_DEVICE");
	g_cur_ordinal = cur ? atoi(cur) & (FAKE_MAX_GPUS - 1) : 0;
	const char *tr = getenv("FAKE_CUDA_TRACE");
	if (tr && *tr)
		g_trace = fopen(tr, "a");
	const char *lp = getenv("FAKE_CUDA_LEDGER");
	if (lp && *lp) {
		int fd = open(lp, O_RDWR | O_CREAT, 0666);
		if (fd >= 0 && ftruncate(fd, 4096) == 0) {
			void *p = mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
			if (p != MAP_FAILED)
				g_ledger = p;
		}
		if (fd >= 0)
			close(fd);
	}
}

static void trace(const char *fmt, ...)
{
	setup_once();
	if (!g_trace)
		return;
	va_list ap;
	va_start(ap, fmt);
	pthread_mutex_lock(&g_mu);
	vfprintf(g_trace, fmt, ap);
	fputc('\n', g_trace);
	fflush(g_trace);
	pthread_mutex_unlock(&g_mu);
	va_end(ap);
}

static uint64_t g_my_phys[FAKE_MAX_GPUS]; /* what this process holds, per physical GPU (under g_mu) */

static int phys_take_on(int gpu, uint64_t bytes)
{
	for (;;) {
		uint64_t cur = __atomic_load_n(&g_ledger->used[gpu], __ATOMIC_SEQ_CST);
		if (cur + bytes > g_total)
			return -1;
		if (__atomic_compare_exchange_n(&g_ledger->used[gpu], &cur, cur + bytes, 0, __ATOMIC_SEQ_CST,
						__ATOMIC_SEQ_CST))
			return 0;
	}
}

static void phys_give_on(int gpu, uint64_t bytes)
{
	__atomic_fetch_sub(&g_ledger->used[gpu], bytes, __ATOMIC_SEQ_CST);
}

/* plain allocations live on the GPU the context is on */
static int phys_take(uint64_t bytes) { return phys_take_on(phys_of(g_cur_ordinal), bytes); }
static void phys_give(uint64_t bytes) { phys_give_on(phys_of(g_cur_ordinal), bytes); }

/* give everything back if the process dies with memory still "on the GPU" */
__attribute__((destructor)) static void on_exit_release(void)
{
	for (int i = 0; i < FAKE_MAX_GPUS; ++i)
		if (g_my_phys[i])
			phys_give_on(i, g_my_phys[i]);
}

/* ------------------------------------------------------ init / device ---- */

CUresult cuInit(unsigned flags)
{
	setup_once();
	trace("cuInit %u", flags);
	g_inited = 1;
	return OK;
}

CUresult cuDriverGetVersion(int *v) { *v = 12090; return OK; }
CUresult cuDeviceGetCount(int *n) { *n = getenv("FAKE_CUDA_DEVICES") ? atoi(getenv("FAKE_CUDA_DEVICES")) : 1; return OK; }
CUresult cuDeviceGet(CUdevice *d, int ord) { *d = ord; return OK; }
CUresult cuDeviceGetName(char *name, int len, CUdevice d) { (void)d; snprintf(name, len, "FAKE H100"); return OK; }
CUresult cuDeviceTotalMem_v2(size_t *b, CUdevice d) { (void)d; setup_once(); *b = g_total; return OK; }
/* the UUID belongs to the physical GPU: two processes that number the GPUs differently agree on it */
CUresult cuDeviceGetUuid_v2(unsigned char uuid[16], CUdevice d)
{
	setup_once();
	if (getenv("FAKE_CUDA_NO_UUID"))
		return E_NOT_FOUND;
	memset(uuid, 0, 16);
	memcpy(uuid, "GPU-FAKE-H100-", 14);
	uuid[15] = (unsigned char)phys_of(d);
	return OK;
}
CUresult cuDeviceGetAttribute(int *v, int attr, CUdevice d)
{
	(void)d;
	switch (attr) {
	case 16: *v = 132; break;  /* SM count */
	case 75: *v = 9; break;    /* cc major */
	case 76: *v = 0; break;    /* cc minor */
	case 102: *v = 1; break;   /* VMM supported */
	default: *v = 1; break;
	}
	return OK;
}
CUresult cuDeviceCanAccessPeer(int *can, CUdevice a, CUdevice b) { *can = (a != b); return OK; }
CUresult cuDevicePrimaryCtxRetain(CUcontext *ctx, CUdevice d) { (void)d; *ctx = &g_ctx_token; return OK; }
CUresult cuDevicePrimaryCtxRelease_v2(CUdevice d) { (void)d; return OK; }
/* One context per process, on FAKE_CUDA_DEVICE -- except that cuCtxCreate for ANOTHER ordinal hands out a
 * second, distinct context (a process that uses two GPUs).  Nothing in here depends on which context is
 * current; the interposer under test does (one swap engine = one context). */
static int g_ctx_token_other;
CUresult cuCtxCreate_v2(CUcontext *ctx, unsigned f, CUdevice d)
{
	(void)f;
	setup_once();
	*ctx = d == g_cur_ordinal ? (void *)&g_ctx_token : (void *)&g_ctx_token_other;
	if (!t_ctx_depth)
		t_ctx_depth = 1;
	t_ctx_stack[t_ctx_depth - 1] = *ctx; /* (the new context becomes current, like in the driver) */
	return OK;
}
CUresult cuCtxGetCurrent(CUcontext *ctx)
{
	*ctx = t_ctx_depth ? t_ctx_stack[t_ctx_depth - 1] : NULL;
	trace("cuCtxGetCurrent");
	return OK;
}
CUresult cuCtxSetCurrent(CUcontext ctx)
{
	trace("cuCtxSetCurrent");
	if (!t_ctx_depth)
		t_ctx_depth = 1;
	t_ctx_stack[t_ctx_depth - 1] = ctx;
	return OK;
}
CUresult cuCtxPushCurrent_v2(CUcontext ctx)
{
	if (t_ctx_depth >= 16)
		return E_INVALID;
	t_ctx_stack[t_ctx_depth++] = ctx;
	return OK;
}
CUresult cuCtxPopCurrent_v2(CUcontext *ctx)
{
	if (!t_ctx_depth)
		return E_INVALID;
	*ctx = t_ctx_stack[--t_ctx_depth];
	return OK;
}
CUresult cuCtxGetDevice(CUdevice *d) { setup_once(); *d = g_cur_ordinal; return OK; }
static CUresult sync_during_capture(const char *what);
CUresult cuCtxSynchronize(void)
{
	CUresult r = sync_during_capture("cuCtxSynchronize");
	if (r)
		return r;
	trace("cuCtxSynchronize");
	return OK;
}
CUresult cuGetErrorString(CUresult e, const char **s) { *s = e == 0 ? "no error" : e == 2 ? "out of memory" : "fake error"; return OK; }
CUresult cuGetErrorName(CUresult e, const char **s) { *s = e == 0 ? "CUDA_SUCCESS" : e == 2 ? "CUDA_ERROR_OUT_OF_MEMORY" : "CUDA_ERROR_FAKE"; return OK; }

/* ------------------------------------------------- plain allocations ----- */

struct plain {
	void *p;
	size_t bytes;
	int device_mem;
	struct plain *next;
};
static struct plain *g_plain;

static CUresult plain_alloc(CUdeviceptr *dptr, size_t bytes, int device_mem)
{
	setup_once();
	if (bytes == 0)
		return E_INVALID;
	if (device_mem && phys_take(bytes) != 0)
		return E_OOM;
	size_t len = (bytes + 4095) & ~4095ull;
	void *p = mmap(NULL, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
	if (p == MAP_FAILED) {
		if (device_mem)
			phys_give(bytes);
		return E_OOM;
	}
	struct plain *n = malloc(sizeof(*n));
	n->p = p;
	n->bytes = bytes;
	n->device_mem = device_mem;
	pthread_mutex_lock(&g_mu);
	n->next = g_plain;
	g_plain = n;
	if (device_mem)
		g_my_phys[phys_of(g_cur_ordinal)] += bytes;
	pthread_mutex_unlock(&g_mu);
	*dptr = (CUdeviceptr)(uintptr_t)p;
	return OK;
}

static CUresult plain_free(CUdeviceptr dptr)
{
	pthread_mutex_lock(&g_mu);
	struct plain **pp = &g_plain;
	while (*pp && (CUdeviceptr)(uintptr_t)(*pp)->p != dptr)
		pp = &(*pp)->next;
	struct plain *n = *pp;
	if (n) {
		*pp = n->next;
		if (n->device_mem)
			g_my_phys[phys_of(g_cur_ordinal)] -= n->bytes;
	}
	pthread_mutex_unlock(&g_mu);
	if (!n)
		return E_INVALID;
	munmap(n->p, (n->bytes + 4095) & ~4095ull);
	if (n->device_mem)
		phys_give(n->bytes);
	free(n);
	return OK;
}

CUresult cuMemAlloc_v2(CUdeviceptr *dptr, size_t bytes)
{
	CUresult r = plain_alloc(dptr, bytes, 1);
	trace("cuMemAlloc %zu -> %d", bytes, r);
	return r;
}
CUresult cuMemAllocManaged(CUdeviceptr *dptr, size_t bytes, unsigned flags)
{
	/* managed memory is pageable: it does not consume the physical ledger */
	CUresult r = plain_alloc(dptr, bytes, 0);
	trace("cuMemAllocManaged %zu %u -> %d", bytes, flags, r);
	return r;
}
CUresult cuMemFree_v2(CUdeviceptr dptr)
{
	CUresult r = plain_free(dptr);
	trace("cuMemFree -> %d", r);
	return r;
}
/* stream-ordered and pitched allocations: plain device memory here (streams run synchronously) */
CUresult cuMemAllocAsync(CUdeviceptr *dptr, size_t bytes, CUstream s)
{
	(void)s;
	CUresult r = plain_alloc(dptr, bytes, 1);
	trace("cuMemAllocAsync %zu -> %d", bytes, r);
	return r;
}
CUresult cuMemAllocFromPoolAsync(CUdeviceptr *dptr, size_t bytes, void *pool, CUstream s)
{
	(void)pool; (void)s;
	CUresult r = plain_alloc(dptr, bytes, 1);
	trace("cuMemAllocFromPoolAsync %zu -> %d", bytes, r);
	return r;
}
CUresult cuMemFreeAsync(CUdeviceptr dptr, CUstream s)
{
	(void)s;
	CUresult r = plain_free(dptr);
	trace("cuMemFreeAsync -> %d", r);
	return r;
}
CUresult cuMemAllocPitch_v2(CUdeviceptr *dptr, size_t *pitch, size_t width, size_t height, unsigned elem)
{
	(void)elem;
	*pitch = (width + 511) & ~(size_t)511;
	CUresult r = plain_alloc(dptr, *pitch * height, 1);
	trace("cuMemAllocPitch %zu x %zu -> %d", width, height, r);
	return r;
}
CUresult cuMemGetInfo_v2(size_t *free_b, size_t *total_b)
{
	setup_once();
	uint64_t used = __atomic_load_n(&g_ledger->used[phys_of(g_cur_ordinal)], __ATOMIC_SEQ_CST);
	*total_b = g_total;
	*free_b = used > g_total ? 0 : g_total - used;
	trace("cuMemGetInfo");
	return OK;
}
CUresult cuMemHostAlloc(void **pp, size_t bytes, unsigned flags)
{
	(void)flags;
	CUdeviceptr d;
	CUresult r = plain_alloc(&d, bytes, 0);
	if (r == OK)
		*pp = (void *)(uintptr_t)d;
	return r;
}
CUresult cuMemFreeHost(void *p) { return plain_free((CUdeviceptr)(uintptr_t)p); }
CUresult cuMemHostGetDevicePointer_v2(CUdeviceptr *d, void *p, unsigned f) { (void)f; *d = (CUdeviceptr)(uintptr_t)p; return OK; }
CUresult cuMemHostRegister_v2(void *p, size_t bytes, unsigned flags) { (void)flags; trace("cuMemHostRegister %zu", bytes); return p ? OK : E_INVALID; }
CUresult cuMemHostUnregister(void *p) { (void)p; return OK; }

/* -------------------------------------------------------------- VMM ------ */

struct phys {
	int fd;
	size_t bytes;
	int live;
	int exported; /* a shareable handle (fd) of it has left this process: the bytes stay charged to the
	               * ledger when we release our reference, whoever imports the fd releases them */
	int gpu;      /* physical GPU whose "HBM" it is (CUmemAllocationProp.location.id, mapped) */
};
#define MAX_PHYS 65536
static struct phys g_phys[MAX_PHYS];

CUresult cuMemGetAllocationGranularity(size_t *g, const void *prop, int opt) { (void)prop; (void)opt; *g = SLAB; return OK; }

CUresult cuMemAddressReserve(CUdeviceptr *ptr, size_t size, size_t align, CUdeviceptr addr, unsigned long long flags)
{
	(void)addr; (void)flags;
	if (size == 0 || (size & (SLAB - 1)))
		return E_INVALID;
	if (align < SLAB)
		align = SLAB;
	void *p = mmap(NULL, size + align, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
	if (p == MAP_FAILED)
		return E_OOM;
	uintptr_t base = ((uintptr_t)p + align - 1) & ~(uintptr_t)(align - 1);
	if (base > (uintptr_t)p)
		munmap(p, base - (uintptr_t)p);
	uintptr_t end = base + size, mend = (uintptr_t)p + size + align;
	if (mend > end)
		munmap((void *)end, mend - end);
	*ptr = base;
	trace("cuMemAddressReserve %zu", size);
	return OK;
}

CUresult cuMemAddressFree(CUdeviceptr ptr, size_t size)
{
	trace("cuMemAddressFree %zu", size);
	return munmap((void *)(uintptr_t)ptr, size) == 0 ? OK : E_INVALID;
}

CUresult cuMemCreate(CUmemGenericAllocationHandle *h, size_t size, const void *prop, unsigned long long flags)
{
	(void)flags;
	setup_once();
	if (size == 0 || (size & (SLAB - 1)))
		return E_INVALID;
	/* CUmemAllocationProp: {type, requestedHandleTypes, location{type, id}, ...}: location.id at byte 12 */
	const int gpu = phys_of(prop ? ((const int *)prop)[3] : g_cur_ordinal);
	if (phys_take_on(gpu, size) != 0) {
		trace("cuMemCreate %zu -> 2", size);
		return E_OOM;
	}
	int fd = memfd_create("fakehbm", 0);
	if (fd < 0 || ftruncate(fd, (off_t)size) != 0) {
		if (fd >= 0)
			close(fd);
		phys_give_on(gpu, size);
		return E_OOM;
	}
	pthread_mutex_lock(&g_mu);
	int slot = -1;
	for (int i = 1; i < MAX_PHYS; ++i)
		if (!g_phys[i].live) {
			slot = i;
			break;
		}
	if (slot > 0) {
		g_phys[slot].fd = fd;
		g_phys[slot].bytes = size;
		g_phys[slot].live = 1;
		g_phys[slot].gpu = gpu;
		g_my_phys[gpu] += size;
	}
	pthread_mutex_unlock(&g_mu);
	if (slot < 0) {
		close(fd);
		phys_give_on(gpu, size);
		return E_OOM;
	}
	*h = (CUmemGenericAllocationHandle)slot;
	trace("cuMemCreate %zu -> 0", size);
	return OK;
}

CUresult cuMemRelease(CUmemGenericAllocationHandle h)
{
	if (h == 0 || h >= MAX_PHYS || !g_phys[h].live)
		return E_INVALID;
	pthread_mutex_lock(&g_mu);
	close(g_phys[h].fd);
	size_t bytes = g_phys[h].bytes;
	int exported = g_phys[h].exported;
	const int gpu = g_phys[h].gpu;
	g_phys[h].live = 0;
	g_phys[h].exported = 0;
	g_my_phys[gpu] -= bytes;
	pthread_mutex_unlock(&g_mu);
	if (!exported)
		phys_give_on(gpu, bytes);
	trace("cuMemRelease %zu", bytes);
	return OK;
}

/* Shareable handles (POSIX fd): the memfd itself.  Physical memory follows the fd: the exporter's
 * release does not return the bytes to the ledger, the importer's does. */
CUresult cuMemExportToShareableHandle(void *out, CUmemGenericAllocationHandle h, int type, unsigned long long flags)
{
	(void)flags;
	if (type != 1 || h == 0 || h >= MAX_PHYS || !g_phys[h].live)
		return E_INVALID;
	int fd = dup(g_phys[h].fd);
	if (fd < 0)
		return E_OOM;
	g_phys[h].exported = 1;
	*(int *)out = fd;
	trace("cuMemExportToShareableHandle %zu", g_phys[h].bytes);
	return OK;
}

CUresult cuMemImportFromShareableHandle(CUmemGenericAllocationHandle *h, void *os_handle, int type)
{
	setup_once();
	int fd = (int)(intptr_t)os_handle;
	struct stat st;
	if (type != 1 || fstat(fd, &st) != 0 || st.st_size == 0)
		return E_INVALID;
	int mine = dup(fd);
	if (mine < 0)
		return E_OOM;
	pthread_mutex_lock(&g_mu);
	int slot = -1;
	for (int i = 1; i < MAX_PHYS; ++i)
		if (!g_phys[i].live) {
			slot = i;
			break;
		}
	if (slot > 0) {
		g_phys[slot].fd = mine;
		g_phys[slot].bytes = (size_t)st.st_size;
		g_phys[slot].live = 1;
		g_phys[slot].exported = 0;
		g_phys[slot].gpu = phys_of(g_cur_ordinal); /* (handles only ever travel between clients of one GPU here) */
		g_my_phys[phys_of(g_cur_ordinal)] += (size_t)st.st_size;
	}
	pthread_mutex_unlock(&g_mu);
	if (slot < 0) {
		close(mine);
		return E_OOM;
	}
	*h = (CUmemGenericAllocationHandle)slot;
	trace("cuMemImportFromShareableHandle %zu", (size_t)st.st_size);
	return OK;
}

CUresult cuMemMap(CUdeviceptr ptr, size_t size, size_t offset, CUmemGenericAllocationHandle h, unsigned long long flags)
{
	(void)flags;
	if (h == 0 || h >= MAX_PHYS || !g_phys[h].live || offset + size > g_phys[h].bytes)
		return E_INVALID;
	void *p = mmap((void *)(uintptr_t)ptr, size, PROT_NONE, MAP_SHARED | MAP_FIXED, g_phys[h].fd, (off_t)offset);
	trace("cuMemMap %zu", size);
	return p == MAP_FAILED ? E_INVALID : OK;
}

CUresult cuMemSetAccess(CUdeviceptr ptr, size_t size, const void *desc, size_t count)
{
	(void)desc; (void)count;
	trace("cuMemSetAccess %zu", size);
	return mprotect((void *)(uintptr_t)ptr, size, PROT_READ | PROT_WRITE) == 0 ? OK : E_INVALID;
}

CUresult cuMemUnmap(CUdeviceptr ptr, size_t size)
{
	void *p = mmap((void *)(uintptr_t)ptr, size, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE | MAP_FIXED, -1, 0);
	trace("cuMemUnmap %zu", size);
	return p == MAP_FAILED ? E_INVALID : OK;
}

/* ----------------------------------------------------- copies / sets ----- */

#define COPY_FN(name, dst_t, src_t, label)                                   \
	CUresult name(dst_t dst, src_t src, size_t n)                        \
	{                                                                    \
		trace(label " %zu", n);                                      \
		memmove((void *)(uintptr_t)dst, (const void *)(uintptr_t)src, n); \
		return OK;                                                   \
	}
#define COPY_FN_ASYNC(name, dst_t, src_t, label)                             \
	CUresult name(dst_t dst, src_t src, size_t n, CUstream s)            \
	{                                                                    \
		(void)s;                                                     \
		trace(label " %zu", n);                                      \
		memmove((void *)(uintptr_t)dst, (const void *)(uintptr_t)src, n); \
		return OK;                                                   \
	}
COPY_FN(cuMemcpy, CUdeviceptr, CUdeviceptr, "cuMemcpy")
COPY_FN_ASYNC(cuMemcpyAsync, CUdeviceptr, CUdeviceptr, "cuMemcpyAsync")
COPY_FN(cuMemcpyHtoD_v2, CUdeviceptr, const void *, "cuMemcpyHtoD")
COPY_FN_ASYNC(cuMemcpyHtoDAsync_v2, CUdeviceptr, const void *, "cuMemcpyHtoDAsync")
COPY_FN(cuMemcpyDtoH_v2, void *, CUdeviceptr, "cuMemcpyDtoH")
COPY_FN_ASYNC(cuMemcpyDtoHAsync_v2, void *, CUdeviceptr, "cuMemcpyDtoHAsync")
COPY_FN(cuMemcpyDtoD_v2, CUdeviceptr, CUdeviceptr, "cuMemcpyDtoD")
COPY_FN_ASYNC(cuMemcpyDtoDAsync_v2, CUdeviceptr, CUdeviceptr, "cuMemcpyDtoDAsync")

CUresult cuMemsetD32Async(CUdeviceptr p, unsigned v, size_t n, CUstream s)
{
	(void)s;
	uint32_t *q = (uint32_t *)(uintptr_t)p;
	for (size_t i = 0; i < n; ++i)
		q[i] = v;
	return OK;
}
CUresult cuMemsetD8_v2(CUdeviceptr p, unsigned char v, size_t n) { trace("cuMemsetD8 %zu", n); memset((void *)(uintptr_t)p, v, n); return OK; }
CUresult cuMemsetD8Async(CUdeviceptr p, unsigned char v, size_t n, CUstream s) { (void)s; trace("cuMemsetD8Async %zu", n); memset((void *)(uintptr_t)p, v, n); return OK; }
CUresult cuMemsetD32_v2(CUdeviceptr p, unsigned v, size_t n) { trace("cuMemsetD32 %zu", n); return cuMemsetD32Async(p, v, n, NULL); }

/* ------------------------------------------------- streams / events ------ */

/* Stream capture, as far as an interposer can tell: a capturing stream records nodes instead of doing
 * work, and a synchronisation while a capture is active is an illegal call that invalidates the capture
 * (CUDA_ERROR_STREAM_CAPTURE_UNSUPPORTED now, ..._INVALIDATED when the capture is ended). */
struct fake_stream { int capture; /* 0 none, 1 active, 2 invalidated */ int pad; };
static struct fake_stream *g_capturing; /* one capture at a time is all the tests need */
CUresult cuStreamCreate(CUstream *s, unsigned f) { (void)f; *s = calloc(1, sizeof(struct fake_stream)); return OK; }
CUresult cuStreamDestroy_v2(CUstream s) { if ((struct fake_stream *)s == g_capturing) g_capturing = NULL; free(s); return OK; }
CUresult cuStreamBeginCapture_v2(CUstream s, int mode)
{
	(void)mode;
	if (!s || g_capturing)
		return E_INVALID;
	g_capturing = s;
	g_capturing->capture = 1;
	trace("cuStreamBeginCapture");
	return OK;
}
CUresult cuStreamIsCapturing(CUstream s, int *status)
{
	*status = s ? ((struct fake_stream *)s)->capture : 0;
	return OK;
}
CUresult cuStreamEndCapture(CUstream s, void **graph)
{
	struct fake_stream *fs = s;
	if (!fs || fs != g_capturing)
		return E_INVALID;
	const int was = fs->capture;
	fs->capture = 0;
	g_capturing = NULL;
	if (graph)
		*graph = was == 1 ? (void *)fs : NULL;
	trace("cuStreamEndCapture -> %d", was == 1 ? 0 : 901);
	return was == 1 ? OK : 901;
}
static CUresult sync_during_capture(const char *what)
{
	if (!g_capturing || g_capturing->capture == 0)
		return OK;
	g_capturing->capture = 2;
	trace("%s during capture -> 900", what);
	return 900;
}
CUresult cuStreamSynchronize(CUstream s)
{
	struct fake_stream *fs = s;
	if (fs && fs->capture)
		return sync_during_capture("cuStreamSynchronize");
	return OK;
}
struct fake_event { struct timespec ts; };
CUresult cuEventCreate(CUevent *e, unsigned f) { (void)f; *e = calloc(1, sizeof(struct fake_event)); return OK; }
CUresult cuEventDestroy_v2(CUevent e) { free(e); return OK; }
CUresult cuEventRecord(CUevent e, CUstream s) { (void)s; clock_gettime(CLOCK_MONOTONIC, &((struct fake_event *)e)->ts); return OK; }
CUresult cuEventSynchronize(CUevent e) { (void)e; return OK; }
CUresult cuEventQuery(CUevent e) { (void)e; return OK; } /* work completes synchronously here */
CUresult cuEventElapsedTime(float *ms, CUevent a, CUevent b)
{
	struct fake_event *x = a, *y = b;
	*ms = (float)((y->ts.tv_sec - x->ts.tv_sec) * 1e3 + (y->ts.tv_nsec - x->ts.tv_nsec) * 1e-6);
	if (*ms <= 0)
		*ms = 1e-3f;
	return OK;
}

/* ------------------------------------------------- modules / launch ------ */

struct fake_fn { char name[64]; };
static struct fake_fn g_fns[32];
static int g_nfns;
static unsigned long g_launches;

CUresult cuModuleLoadData(CUmodule *m, const void *image)
{
	if (getenv("FAKE_CUDA_NO_BINARY")) { /* "this GPU is not sm_90a": CUDA_ERROR_NO_BINARY_FOR_GPU */
		trace("cuModuleLoadData -> 209");
		return 209;
	}
	*m = (void *)image;
	trace("cuModuleLoadData");
	return image ? OK : E_INVALID;
}
CUresult cuModuleUnload(CUmodule m) { (void)m; return OK; }
CUresult cuModuleGetFunction(CUfunction *f, CUmodule m, const char *name)
{
	(void)m;
	pthread_mutex_lock(&g_mu);
	int i;
	for (i = 0; i < g_nfns; ++i)
		if (!strcmp(g_fns[i].name, name))
			break;
	if (i == g_nfns && g_nfns < 32) {
		snprintf(g_fns[i].name, sizeof(g_fns[i].name), "%s", name);
		g_nfns++;
	}
	pthread_mutex_unlock(&g_mu);
	if (i >= 32)
		return E_NOT_FOUND;
	*f = &g_fns[i];
	return OK;
}
CUresult cuFuncSetAttribute(CUfunction f, int a, int v) { (void)f; (void)a; (void)v; return OK; }

struct desc { uint64_t src, dst, bytes, tag; };

static uint64_t pattern(uint64_t i, uint64_t seed)
{
	uint64_t z = i + seed * 0x9E3779B97F4A7C15ull + 0x9E3779B97F4A7C15ull;
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

CUresult cuLaunchKernel(CUfunction f, unsigned gx, unsigned gy, unsigned gz, unsigned bx, unsigned by, unsigned bz,
			unsigned smem, CUstream s, void **params, void **extra)
{
	(void)gy; (void)gz; (void)by; (void)bz; (void)s; (void)extra;
	__atomic_fetch_add(&g_launches, 1, __ATOMIC_RELAXED);
	int ours = 0;
	for (int i = 0; i < g_nfns; ++i)
		ours |= (f == (CUfunction)&g_fns[i]);
	if (!ours) {
		trace("cuLaunchKernel");
		return OK;
	}
	const char *name = ((struct fake_fn *)f)->name;
	trace("cuLaunchKernel %s grid=%u block=%u smem=%u", name, gx, bx, smem);
	if (!strcmp(name, "nvs_slab_copy_tma") || !strcmp(name, "nvs_slab_copy_ldg")) {
		const struct desc *d = *(const struct desc **)params[0];
		uint32_t n = *(uint32_t *)params[1];
		uint32_t *counter = *(uint32_t **)params[2];
		if (*counter != 0)
			return 999; /* the engine must hand every launch a zeroed counter */
		for (uint32_t i = 0; i < n; ++i)
			memcpy((void *)(uintptr_t)d[i].dst, (const void *)(uintptr_t)d[i].src, d[i].bytes);
		*counter = n + gx; /* what the real kernel leaves behind: every CTA over-increments once */
		return OK;
	}
	if (!strcmp(name, "nvs_slab_scan")) {
		const struct desc *d = *(const struct desc **)params[0];
		uint32_t n = *(uint32_t *)params[1];
		uint32_t *counter = *(uint32_t **)params[2];
		struct { uint64_t value, is_const, h0, h1; } *out = *(void **)params[3];
		uint32_t want_hash = *(uint32_t *)params[4];
		if (*counter != 0 || bx != 256)
			return 999;
		for (uint32_t i = 0; i < n; ++i) {
			const uint64_t *p = (const uint64_t *)(uintptr_t)d[i].src;
			uint64_t words = d[i].bytes / 8, k = 1, h[2] = {0, 0};
			if (d[i].dst) {
				/* fused copy + hash: in the real kernel every lane hashes the very vector it stores, so the
				 * result describes what LANDED in dst even if the source is being written meanwhile
				 * (application threads, here) -- emulated by looking at the copy, not at the source again */
				memcpy((void *)(uintptr_t)d[i].dst, p, d[i].bytes & ~15ull);
				p = (const uint64_t *)(uintptr_t)d[i].dst;
			}
			while (k < words && p[k] == p[0])
				++k;
			out[i].value = p[0];
			out[i].is_const = (k == words) && (d[i].bytes & 15) == 0;
			if (want_hash || d[i].dst)
				slab_hash_ref(p, d[i].bytes, h);
			out[i].h0 = h[0];
			out[i].h1 = h[1];
		}
		*counter = n + gx;
		return OK;
	}
	if (!strcmp(name, "nvs_slab_splat")) {
		const struct desc *d = *(const struct desc **)params[0];
		uint32_t n = *(uint32_t *)params[1];
		uint32_t *counter = *(uint32_t **)params[2];
		if (*counter != 0)
			return 999;
		for (uint32_t i = 0; i < n; ++i) {
			uint64_t *q = (uint64_t *)(uintptr_t)d[i].dst;
			for (uint64_t k = 0; k < d[i].bytes / 8; ++k)
				q[k] = d[i].src;
		}
		*counter = n + gx;
		return OK;
	}
	if (!strcmp(name, "nvs_slab_fill")) {
		uint64_t *p = *(uint64_t **)params[0];
		uint64_t n = *(uint64_t *)params[1], first = *(uint64_t *)params[2], seed = *(uint64_t *)params[3];
		for (uint64_t i = 0; i < n; ++i)
			p[i] = pattern(first + i, seed);
		return OK;
	}
	if (!strcmp(name, "nvs_slab_verify")) {
		const uint64_t *p = *(const uint64_t **)params[0];
		uint64_t n = *(uint64_t *)params[1], first = *(uint64_t *)params[2], seed = *(uint64_t *)params[3];
		unsigned long long *out = *(unsigned long long **)params[4];
		unsigned long long bad = 0;
		for (uint64_t i = 0; i < n; ++i)
			bad += p[i] != pattern(first + i, seed);
		*out += bad;
		return OK;
	}
	return OK;
}

unsigned long fake_cuda_launch_count(void) { return g_launches; }
uint64_t fake_cuda_phys_used(void) { setup_once(); return __atomic_load_n(&g_ledger->used[phys_of(g_cur_ordinal)], __ATOMIC_SEQ_CST); }
uint64_t fake_cuda_phys_used_on(int ordinal) { setup_once(); return __atomic_load_n(&g_ledger->used[phys_of(ordinal)], __ATOMIC_SEQ_CST); }

/* -------------------------------------------------- cuGetProcAddress ----- */

static void *lookup_self(const char *symbol)
{
	static const char *suffixes[] = {"", "_v2", "_v3", NULL};
	char buf[160];
	Dl_info info;
	void *self = NULL;
	if (dladdr((void *)&cuInit, &info) && info.dli_fname)
		self = dlopen(info.dli_fname, RTLD_NOW | RTLD_NOLOAD);
	for (int i = 0; suffixes[i]; ++i) {
		snprintf(buf, sizeof(buf), "%s%s", symbol, suffixes[i]);
		void *p = self ? dlsym(self, buf) : NULL;
		if (p && i == 0) {
			/* prefer the versioned spelling when both exist */
			char b2[160];
			snprintf(b2, sizeof(b2), "%s_v2", symbol);
			void *p2 = dlsym(self, b2);
			if (p2)
				return p2;
		}
		if (p)
			return p;
	}
	return NULL;
}

CUresult cuGetProcAddress(const char *symbol, void **pfn, int ver, uint64_t flags)
{
	(void)ver; (void)flags;
	*pfn = lookup_self(symbol);
	trace("cuGetProcAddress %s", symbol);
	return *pfn ? OK : E_NOT_FOUND;
}

CUresult cuGetProcAddress_v2(const char *symbol, void **pfn, int ver, uint64_t flags, int *status)
{
	(void)ver; (void)flags;
	*pfn = lookup_self(symbol);
	if (status)
		*status = *pfn ? 0 : 1;
	trace("cuGetProcAddress_v2 %s", symbol);
	return OK;
}
