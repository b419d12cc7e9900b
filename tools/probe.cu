/*
 * probe.cu -- one-shot measurement of every GPU / driver constant the swap
 * engine's design depends on (DESIGN.md cites the numbers this prints):
 *
 *   A  device + host facts (SMs, HBM, VMM granularity, host RAM, cores)
 *   B  VMM cost: cuMemCreate / cuMemMap / cuMemSetAccess / cuMemUnmap /
 *      cuMemRelease as a function of the mapping-chunk size
 *   C  pinned-host provisioning rate (cuMemHostAlloc, cuMemHostRegister)
 *   D  slab copy bandwidth HBM<->pinned host and HBM<->HBM: copy engines
 *      (control), nvs_slab_copy_tma, nvs_slab_copy_ldg, swept over grid size
 *      and ring geometry, single direction and full duplex, each verified
 *      bit-exact against the position-dependent pattern
 *   E  the reference's mechanism on this box: cuMemAllocManaged fault-driven
 *      and prefetch-driven migration bandwidth
 *   F  peer-HBM tier (only when >= 2 devices are visible)
 *
 * Output: one JSON object per line on stdout ("PROBE {...}").
 * Build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo \
 *              -o tools/probe tools/probe.cu -lcuda
 * This is a measurement tool, not part of the product path.
 */
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <time.h>
#include <unistd.h>
#include <sys/mman.h>
#include <pthread.h>
#include <vector>
#include <algorithm>

#include "../nvshare_b200/csrc/slab_copy.cu"

#define MiB (1ull << 20)
#define GiB (1ull << 30)

static double now_s(void)
{
	struct timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec + ts.tv_nsec * 1e-9;
}

#define CU(call)                                                                       \
	do {                                                                           \
		CUresult _r = (call);                                                  \
		if (_r != CUDA_SUCCESS) {                                              \
			const char *_n = "?";                                          \
			cuGetErrorName(_r, &_n);                                       \
			printf("PROBE {\"error\":\"%s\",\"rc\":%d,\"name\":\"%s\",\"line\":%d}\n", \
			       #call, (int)_r, _n, __LINE__);                          \
			fflush(stdout);                                                \
			return -1;                                                     \
		}                                                                      \
	} while (0)

#define RT(call)                                                                       \
	do {                                                                           \
		cudaError_t _r = (call);                                               \
		if (_r != cudaSuccess) {                                               \
			printf("PROBE {\"error\":\"%s\",\"rc\":%d,\"name\":\"%s\",\"line\":%d}\n", \
			       #call, (int)_r, cudaGetErrorName(_r), __LINE__);        \
			fflush(stdout);                                                \
			return -1;                                                     \
		}                                                                      \
	} while (0)

static int g_dev = 0;
static int g_sms = 0;
static size_t g_scale_gib = 8; /* working-set size for sections D/E/F */

/* --------------------------------------------------------------- A ------ */
static int section_a(void)
{
	CUdevice dev;
	CU(cuDeviceGet(&dev, g_dev));
	char name[128];
	CU(cuDeviceGetName(name, sizeof name, dev));
	size_t total = 0, freeb = 0;
	CU(cuMemGetInfo(&freeb, &total));
	int sms, vmm, pageable, hostreg, ce, cc_major, cc_minor, managed, conc_managed, l2, fd_ok,
		gdr, unified, map_host;
	CU(cuDeviceGetAttribute(&sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev));
	CU(cuDeviceGetAttribute(&vmm, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, dev));
	CU(cuDeviceGetAttribute(&pageable, CU_DEVICE_ATTRIBUTE_PAGEABLE_MEMORY_ACCESS, dev));
	CU(cuDeviceGetAttribute(&hostreg, CU_DEVICE_ATTRIBUTE_HOST_REGISTER_SUPPORTED, dev));
	CU(cuDeviceGetAttribute(&ce, CU_DEVICE_ATTRIBUTE_ASYNC_ENGINE_COUNT, dev));
	CU(cuDeviceGetAttribute(&cc_major, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR, dev));
	CU(cuDeviceGetAttribute(&cc_minor, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR, dev));
	CU(cuDeviceGetAttribute(&managed, CU_DEVICE_ATTRIBUTE_MANAGED_MEMORY, dev));
	CU(cuDeviceGetAttribute(&conc_managed, CU_DEVICE_ATTRIBUTE_CONCURRENT_MANAGED_ACCESS, dev));
	CU(cuDeviceGetAttribute(&l2, CU_DEVICE_ATTRIBUTE_L2_CACHE_SIZE, dev));
	CU(cuDeviceGetAttribute(&fd_ok, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev));
	CU(cuDeviceGetAttribute(&gdr, CU_DEVICE_ATTRIBUTE_GPU_DIRECT_RDMA_SUPPORTED, dev));
	CU(cuDeviceGetAttribute(&unified, CU_DEVICE_ATTRIBUTE_UNIFIED_ADDRESSING, dev));
	CU(cuDeviceGetAttribute(&map_host, CU_DEVICE_ATTRIBUTE_CAN_MAP_HOST_MEMORY, dev));
	g_sms = sms;

	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof prop);
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = g_dev;
	size_t gmin = 0, grec = 0;
	CU(cuMemGetAllocationGranularity(&gmin, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
	CU(cuMemGetAllocationGranularity(&grec, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
	int ndev = 0;
	CU(cuDeviceGetCount(&ndev));
	int drv = 0;
	CU(cuDriverGetVersion(&drv));
	long ncpu = sysconf(_SC_NPROCESSORS_ONLN);
	long pages = sysconf(_SC_PHYS_PAGES), psz = sysconf(_SC_PAGE_SIZE);
	printf("PROBE {\"section\":\"A\",\"name\":\"%s\",\"cc\":\"%d.%d\",\"sms\":%d,\"hbm_total\":%zu,"
	       "\"hbm_free\":%zu,\"vmm\":%d,\"gran_min\":%zu,\"gran_rec\":%zu,\"pageable_access\":%d,"
	       "\"host_register\":%d,\"async_engines\":%d,\"managed\":%d,\"concurrent_managed\":%d,"
	       "\"l2_bytes\":%d,\"posix_fd_handles\":%d,\"gdr\":%d,\"uva\":%d,\"map_host\":%d,"
	       "\"n_devices\":%d,\"driver\":%d,\"host_cpus\":%ld,\"host_ram_bytes\":%lld}\n",
	       name, cc_major, cc_minor, sms, total, freeb, vmm, gmin, grec, pageable, hostreg, ce,
	       managed, conc_managed, l2, fd_ok, gdr, unified, map_host, ndev, drv, ncpu,
	       (long long)pages * psz);
	fflush(stdout);
	return 0;
}

/* --------------------------------------------------------------- B ------ */
static int vmm_one(size_t chunk, size_t total)
{
	const size_t n = total / chunk;
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof prop);
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = g_dev;
	CUmemAccessDesc acc;
	memset(&acc, 0, sizeof acc);
	acc.location = prop.location;
	acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;

	CUdeviceptr va = 0;
	double t0 = now_s();
	CU(cuMemAddressReserve(&va, total, 0, 0, 0));
	double t_res = now_s() - t0;
	std::vector<CUmemGenericAllocationHandle> h(n);

	t0 = now_s();
	for (size_t i = 0; i < n; ++i)
		CU(cuMemCreate(&h[i], chunk, &prop, 0));
	double t_create = now_s() - t0;
	t0 = now_s();
	for (size_t i = 0; i < n; ++i)
		CU(cuMemMap(va + i * chunk, chunk, 0, h[i], 0));
	double t_map = now_s() - t0;
	t0 = now_s();
	CU(cuMemSetAccess(va, total, &acc, 1));
	double t_acc_one = now_s() - t0;
	/* touch it so that lazily-built page tables (if any) are paid for here */
	RT(cudaMemset((void *)va, 1, total));
	RT(cudaDeviceSynchronize());
	t0 = now_s();
	for (size_t i = 0; i < n; ++i)
		CU(cuMemUnmap(va + i * chunk, chunk));
	double t_unmap = now_s() - t0;
	t0 = now_s();
	for (size_t i = 0; i < n; ++i)
		CU(cuMemRelease(h[i]));
	double t_release = now_s() - t0;

	/* second pass: per-chunk create+map+setaccess interleaved (the fetch order) */
	t0 = now_s();
	for (size_t i = 0; i < n; ++i) {
		CU(cuMemCreate(&h[i], chunk, &prop, 0));
		CU(cuMemMap(va + i * chunk, chunk, 0, h[i], 0));
		CU(cuMemSetAccess(va + i * chunk, chunk, &acc, 1));
	}
	double t_fetch_order = now_s() - t0;
	t0 = now_s();
	for (size_t i = 0; i < n; ++i) {
		CU(cuMemUnmap(va + i * chunk, chunk));
		CU(cuMemRelease(h[i]));
	}
	double t_evict_order = now_s() - t0;
	CU(cuMemAddressFree(va, total));

	printf("PROBE {\"section\":\"B\",\"chunk_mib\":%llu,\"total_gib\":%.1f,\"n\":%zu,"
	       "\"reserve_ms\":%.3f,\"create_us_per\":%.1f,\"map_us_per\":%.1f,\"setaccess_whole_ms\":%.3f,"
	       "\"unmap_us_per\":%.1f,\"release_us_per\":%.1f,\"fetch_order_ms\":%.2f,"
	       "\"evict_order_ms\":%.2f,\"map_GBps\":%.1f,\"unmap_GBps\":%.1f}\n",
	       chunk / MiB, (double)total / GiB, n, t_res * 1e3, t_create * 1e6 / n, t_map * 1e6 / n,
	       t_acc_one * 1e3, t_unmap * 1e6 / n, t_release * 1e6 / n, t_fetch_order * 1e3,
	       t_evict_order * 1e3, total / 1e9 / t_fetch_order, total / 1e9 / t_evict_order);
	fflush(stdout);
	return 0;
}

static int section_b(void)
{
	const size_t total = 8 * GiB;
	const size_t chunks[] = {2 * MiB, 8 * MiB, 32 * MiB, 64 * MiB, 256 * MiB, 1024 * MiB};
	for (size_t c : chunks)
		if (vmm_one(c, total) != 0)
			return -1;
	return 0;
}

/* --------------------------------------------------------------- C ------ */
static int section_c(void)
{
	const size_t sizes[] = {256 * MiB, 1 * GiB, 4 * GiB};
	for (size_t sz : sizes) {
		void *p = NULL;
		double t0 = now_s();
		CU(cuMemHostAlloc(&p, sz, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
		double t_alloc = now_s() - t0;
		t0 = now_s();
		memset(p, 0x5a, sz);
		double t_touch = now_s() - t0;
		t0 = now_s();
		CU(cuMemFreeHost(p));
		double t_free = now_s() - t0;
		printf("PROBE {\"section\":\"C\",\"how\":\"cuMemHostAlloc\",\"bytes\":%zu,\"alloc_ms\":%.1f,"
		       "\"alloc_GBps\":%.2f,\"first_touch_GBps\":%.2f,\"free_ms\":%.1f}\n",
		       sz, t_alloc * 1e3, sz / 1e9 / t_alloc, sz / 1e9 / t_touch, t_free * 1e3);
		fflush(stdout);
	}
	/* register path: mmap + populate (optionally THP) + cuMemHostRegister */
	for (int thp = 0; thp < 2; ++thp) {
		const size_t sz = 4 * GiB;
		void *p = mmap(NULL, sz, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
		if (p == MAP_FAILED) {
			printf("PROBE {\"section\":\"C\",\"error\":\"mmap\"}\n");
			continue;
		}
		if (thp)
			madvise(p, sz, MADV_HUGEPAGE);
		double t0 = now_s();
		memset(p, 1, sz);
		double t_touch = now_s() - t0;
		t0 = now_s();
		CUresult r = cuMemHostRegister(p, sz, CU_MEMHOSTREGISTER_PORTABLE | CU_MEMHOSTREGISTER_DEVICEMAP);
		double t_reg = now_s() - t0;
		printf("PROBE {\"section\":\"C\",\"how\":\"mmap+register\",\"thp\":%d,\"bytes\":%zu,\"rc\":%d,"
		       "\"touch_GBps\":%.2f,\"register_ms\":%.1f,\"register_GBps\":%.2f}\n",
		       thp, sz, (int)r, sz / 1e9 / t_touch, t_reg * 1e3, sz / 1e9 / t_reg);
		fflush(stdout);
		if (r == CUDA_SUCCESS)
			cuMemHostUnregister(p);
		munmap(p, sz);
	}
	return 0;
}

/* --------------------------------------------------------------- D ------ */
struct Bufs {
	CUdeviceptr dev_a, dev_b; /* HBM */
	uint8_t *host_a, *host_b; /* pinned, device-mapped (UVA: same address on device) */
	nvs_copy_desc *descs_h;   /* pinned staging for descriptor lists */
	nvs_copy_desc *descs_d[2];
	uint32_t *counters;       /* device */
	unsigned long long *mism; /* device */
	size_t bytes;
	size_t n_slabs;
	cudaStream_t st[2];
	cudaEvent_t ev[4];
};

static int fill(const Bufs &b, CUdeviceptr p, uint64_t seed)
{
	nvs_slab_fill<<<g_sms * 8, 256>>>((uint64_t *)p, b.bytes / 8, 0, seed);
	RT(cudaGetLastError());
	RT(cudaDeviceSynchronize());
	return 0;
}

static long long verify(const Bufs &b, CUdeviceptr p, uint64_t seed)
{
	if (cudaMemset(b.mism, 0, 8) != cudaSuccess)
		return -2;
	nvs_slab_verify<<<g_sms * 8, 256>>>((const uint64_t *)p, b.bytes / 8, 0, seed, b.mism);
	if (cudaGetLastError() != cudaSuccess)
		return -3;
	unsigned long long m = 0;
	if (cudaMemcpy(&m, b.mism, 8, cudaMemcpyDeviceToHost) != cudaSuccess)
		return -4;
	return (long long)m;
}

static void build_descs(const Bufs &b, int which, uint64_t src, uint64_t dst)
{
	/* descriptor i moves slab perm(i): a fixed odd-multiplier permutation so
	 * consecutive descriptors are not address-adjacent (worst case for DMA
	 * coalescing, and what an LRU-ordered eviction looks like) */
	nvs_copy_desc *h = b.descs_h + (size_t)which * b.n_slabs;
	const bool pow2 = (b.n_slabs & (b.n_slabs - 1)) == 0;
	for (size_t i = 0; i < b.n_slabs; ++i) {
		/* odd multiplier modulo a power of two is a bijection */
		const size_t s = pow2 ? ((i * 2654435761ull) & (b.n_slabs - 1)) : i;
		h[i].src = src + s * NVS_SLAB_BYTES;
		h[i].dst = dst + s * NVS_SLAB_BYTES;
		h[i].bytes = NVS_SLAB_BYTES;
		h[i].tag = s;
	}
	cudaMemcpy(b.descs_d[which], h, b.n_slabs * sizeof(nvs_copy_desc), cudaMemcpyHostToDevice);
}

struct Geo {
	int variant; /* NVS_COPY_* */
	int grid;
	int warps;  /* TMA: warps per CTA; LDG: threads/32 */
	int stages; /* TMA */
	int tile;   /* TMA tile bytes */
};

static int launch_copy(const Bufs &b, int which, const Geo &g, cudaStream_t st)
{
	uint32_t *ctr = b.counters + which;
	RT(cudaMemsetAsync(ctr, 0, 4, st));
	if (g.variant == NVS_COPY_TMA) {
		size_t smem = (size_t)g.warps * g.stages * g.tile;
		nvs_slab_copy_tma<<<g.grid, 32 * g.warps, smem, st>>>(b.descs_d[which], (uint32_t)b.n_slabs,
								      ctr, g.tile, g.stages);
	} else if (g.variant == NVS_COPY_LDG) {
		nvs_slab_copy_ldg<<<g.grid, 32 * g.warps, 0, st>>>(b.descs_d[which], (uint32_t)b.n_slabs, ctr);
	} else {
		const nvs_copy_desc *h = b.descs_h + (size_t)which * b.n_slabs;
		for (size_t i = 0; i < b.n_slabs; ++i)
			CU(cuMemcpyAsync(h[i].dst, h[i].src, h[i].bytes, st));
	}
	RT(cudaGetLastError());
	return 0;
}

/* time `reps` repetitions of one direction (or two concurrently when duplex) */
static int time_copy(const Bufs &b, const Geo &g, bool duplex, int reps, double *ms_out, double *issue_ms)
{
	/* warm-up */
	if (launch_copy(b, 0, g, b.st[0]))
		return -1;
	if (duplex && launch_copy(b, 1, g, b.st[1]))
		return -1;
	RT(cudaDeviceSynchronize());
	double best = 1e30, best_issue = 0;
	for (int r = 0; r < reps; ++r) {
		RT(cudaEventRecord(b.ev[0], b.st[0]));
		if (duplex) {
			RT(cudaStreamWaitEvent(b.st[1], b.ev[0], 0));
		}
		double t0 = now_s();
		if (launch_copy(b, 0, g, b.st[0]))
			return -1;
		if (duplex && launch_copy(b, 1, g, b.st[1]))
			return -1;
		double t_issue = (now_s() - t0) * 1e3;
		if (duplex) {
			RT(cudaEventRecord(b.ev[2], b.st[1]));
			RT(cudaStreamWaitEvent(b.st[0], b.ev[2], 0));
		}
		RT(cudaEventRecord(b.ev[1], b.st[0]));
		RT(cudaEventSynchronize(b.ev[1]));
		float ms = 0;
		RT(cudaEventElapsedTime(&ms, b.ev[0], b.ev[1]));
		if (ms < best) {
			best = ms;
			best_issue = t_issue;
		}
	}
	*ms_out = best;
	*issue_ms = best_issue;
	return 0;
}

static const char *vname(int v)
{
	return v == NVS_COPY_TMA ? "tma" : v == NVS_COPY_LDG ? "ldg" : "ce";
}

static int run_case(Bufs &b, const char *dir, const Geo &g, bool duplex, bool check)
{
	/* directions: "d2h": dev_a -> host_a ; "h2d": host_a -> dev_a ; "d2d": dev_a -> dev_b
	 * duplex: d2h (dev_a->host_a) on stream 0 + h2d (host_b->dev_b) on stream 1 */
	uint64_t src0, dst0;
	if (!strcmp(dir, "d2h")) {
		src0 = b.dev_a;
		dst0 = (uint64_t)b.host_a;
	} else if (!strcmp(dir, "h2d")) {
		src0 = (uint64_t)b.host_a;
		dst0 = b.dev_a;
	} else {
		src0 = b.dev_a;
		dst0 = b.dev_b;
	}
	build_descs(b, 0, src0, dst0);
	if (duplex)
		build_descs(b, 1, (uint64_t)b.host_b, b.dev_b);
	if (check) {
		/* poison the destination(s) so a skipped slab cannot pass */
		nvs_slab_fill<<<g_sms * 8, 256>>>((uint64_t *)dst0, b.bytes / 8, 0, 99);
		if (duplex)
			nvs_slab_fill<<<g_sms * 8, 256>>>((uint64_t *)b.dev_b, b.bytes / 8, 0, 99);
		RT(cudaDeviceSynchronize());
	}
	double ms = 0, issue = 0;
	if (time_copy(b, g, duplex, 2, &ms, &issue))
		return -1;
	long long bad = -1;
	if (check) {
		/* destination must now carry the source's pattern (seed 1 lives in dev_a /
		 * host_a after the d2h pass; seed 2 in host_b) */
		bad = verify(b, dst0, 1);
		if (duplex) {
			long long bad2 = verify(b, b.dev_b, 2);
			bad = (bad < 0 || bad2 < 0) ? -1 : bad + bad2;
		}
	}
	const double gb = b.bytes / 1e9;
	printf("PROBE {\"section\":\"D\",\"dir\":\"%s%s\",\"variant\":\"%s\",\"grid\":%d,\"warps\":%d,"
	       "\"stages\":%d,\"tile\":%d,\"bytes_per_dir\":%zu,\"ms\":%.3f,\"GBps_per_dir\":%.2f,"
	       "\"GBps_total\":%.2f,\"issue_ms\":%.3f,\"mismatches\":%lld}\n",
	       dir, duplex ? "+h2d" : "", vname(g.variant), g.grid, g.warps, g.stages, g.tile, b.bytes,
	       ms, gb / (ms * 1e-3), (duplex ? 2 : 1) * gb / (ms * 1e-3), issue, bad);
	fflush(stdout);
	return bad > 0 ? -1 : 0;
}

static int section_d(void)
{
	Bufs b;
	memset(&b, 0, sizeof b);
	b.bytes = g_scale_gib * GiB / 2; /* 4 GiB per buffer by default */
	b.n_slabs = b.bytes / NVS_SLAB_BYTES;
	CU(cuMemAlloc(&b.dev_a, b.bytes));
	CU(cuMemAlloc(&b.dev_b, b.bytes));
	CU(cuMemHostAlloc((void **)&b.host_a, b.bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	CU(cuMemHostAlloc((void **)&b.host_b, b.bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	CU(cuMemHostAlloc((void **)&b.descs_h, 2 * b.n_slabs * sizeof(nvs_copy_desc), CU_MEMHOSTALLOC_PORTABLE));
	RT(cudaMalloc(&b.descs_d[0], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.descs_d[1], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.counters, 64));
	RT(cudaMalloc(&b.mism, 8));
	for (int i = 0; i < 2; ++i)
		RT(cudaStreamCreateWithFlags(&b.st[i], cudaStreamNonBlocking));
	for (int i = 0; i < 4; ++i)
		RT(cudaEventCreate(&b.ev[i]));
	RT(cudaFuncSetAttribute(nvs_slab_copy_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));

	/* device pointer of mapped host memory must equal the host pointer (UVA) */
	CUdeviceptr dp = 0;
	CU(cuMemHostGetDevicePointer(&dp, b.host_a, 0));
	printf("PROBE {\"section\":\"D\",\"uva_host_eq_dev\":%d}\n", dp == (CUdeviceptr)b.host_a);

	if (fill(b, b.dev_a, 1))
		return -1;
	/* host_b carries pattern seed 2 (written by the GPU through the mapping) */
	if (fill(b, (CUdeviceptr)b.host_b, 2))
		return -1;
	memset(b.host_a, 0, b.bytes);

	/* 0. smoke: one tiny TMA launch first, so a hang shows up here */
	{
		Geo g = {NVS_COPY_TMA, 1, 1, 2, 16384};
		size_t keep = b.n_slabs, keepb = b.bytes;
		b.n_slabs = 2;
		b.bytes = 2 * NVS_SLAB_BYTES;
		printf("PROBE {\"section\":\"D\",\"note\":\"tma smoke start\"}\n");
		fflush(stdout);
		int rc = run_case(b, "d2d", g, false, true);
		b.n_slabs = keep;
		b.bytes = keepb;
		if (rc)
			return -1;
	}

	/* 1. copy-engine control */
	{
		Geo g = {NVS_COPY_CE, 0, 0, 0, 0};
		if (run_case(b, "d2h", g, false, true)) return -1;
		if (run_case(b, "h2d", g, false, true)) return -1;
		if (run_case(b, "d2h", g, true, true)) return -1;
		if (run_case(b, "d2d", g, false, true)) return -1;
		/* one big call instead of 2 MiB pieces */
		double t0;
		RT(cudaEventRecord(b.ev[0], b.st[0]));
		t0 = now_s();
		CU(cuMemcpyAsync((CUdeviceptr)b.host_a, b.dev_a, b.bytes, b.st[0]));
		RT(cudaEventRecord(b.ev[1], b.st[0]));
		RT(cudaEventSynchronize(b.ev[1]));
		(void)t0;
		float ms;
		RT(cudaEventElapsedTime(&ms, b.ev[0], b.ev[1]));
		printf("PROBE {\"section\":\"D\",\"dir\":\"d2h\",\"variant\":\"ce_onecall\",\"ms\":%.3f,\"GBps_per_dir\":%.2f}\n",
		       ms, b.bytes / 1e9 / (ms * 1e-3));
		RT(cudaEventRecord(b.ev[0], b.st[0]));
		CU(cuMemcpyAsync(b.dev_a, (CUdeviceptr)b.host_a, b.bytes, b.st[0]));
		RT(cudaEventRecord(b.ev[1], b.st[0]));
		RT(cudaEventSynchronize(b.ev[1]));
		RT(cudaEventElapsedTime(&ms, b.ev[0], b.ev[1]));
		printf("PROBE {\"section\":\"D\",\"dir\":\"h2d\",\"variant\":\"ce_onecall\",\"ms\":%.3f,\"GBps_per_dir\":%.2f}\n",
		       ms, b.bytes / 1e9 / (ms * 1e-3));
		fflush(stdout);
	}

	/* 2. TMA sweep */
	const int grids[] = {1, 2, 4, 8, 16, 32, 66, 132};
	const Geo shapes[] = {
		{NVS_COPY_TMA, 0, 1, 6, 32768},
		{NVS_COPY_TMA, 0, 4, 3, 16384},
		{NVS_COPY_TMA, 0, 2, 3, 32768},
		{NVS_COPY_TMA, 0, 1, 3, 65536},
		{NVS_COPY_TMA, 0, 8, 3, 8192},
	};
	for (const Geo &sh : shapes) {
		for (int grid : grids) {
			Geo g = sh;
			g.grid = grid;
			bool check = (grid == 8 || grid == 132);
			if (run_case(b, "d2h", g, false, check)) return -1;
			if (run_case(b, "h2d", g, false, check)) return -1;
			if (grid >= 2) {
				Geo gh = g;
				gh.grid = grid / 2;
				if (run_case(b, "d2h", gh, true, check)) return -1;
			}
			if (grid >= 32)
				if (run_case(b, "d2d", g, false, check)) return -1;
		}
	}
	/* 3. LDG sweep */
	for (int warps : {8, 16}) {
		for (int grid : grids) {
			Geo g = {NVS_COPY_LDG, grid, warps, 0, 0};
			bool check = (grid == 8 || grid == 132);
			if (run_case(b, "d2h", g, false, check)) return -1;
			if (run_case(b, "h2d", g, false, check)) return -1;
			if (grid >= 2) {
				Geo gh = g;
				gh.grid = grid / 2;
				if (run_case(b, "d2h", gh, true, check)) return -1;
			}
			if (grid >= 32)
				if (run_case(b, "d2d", g, false, check)) return -1;
		}
	}
	/* D2D at 2 and 4 CTAs/SM for the HBM roofline */
	for (int mult : {2, 4}) {
		Geo g = {NVS_COPY_LDG, g_sms * mult, 8, 0, 0};
		if (run_case(b, "d2d", g, false, true)) return -1;
		Geo t = {NVS_COPY_TMA, g_sms * mult, 1, 3, 16384};
		if (run_case(b, "d2d", t, false, true)) return -1;
	}

	cuMemFree(b.dev_a);
	cuMemFree(b.dev_b);
	cuMemFreeHost(b.host_a);
	cuMemFreeHost(b.host_b);
	cuMemFreeHost(b.descs_h);
	cudaFree(b.descs_d[0]);
	cudaFree(b.descs_d[1]);
	cudaFree(b.counters);
	cudaFree(b.mism);
	return 0;
}

/* --------------------------------------------------------------- E ------ */
__global__ void touch_sum(const uint64_t *p, uint64_t n_words, unsigned long long *out)
{
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	unsigned long long acc = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride)
		acc += p[i];
	if (acc == 0x1234567)
		atomicAdd(out, acc);
}

static int section_e(void)
{
	const size_t bytes = g_scale_gib * GiB / 2;
	CUdeviceptr m = 0;
	CU(cuMemAllocManaged(&m, bytes, CU_MEM_ATTACH_GLOBAL));
	unsigned long long *out;
	RT(cudaMalloc(&out, 8));
	cudaEvent_t e0, e1;
	RT(cudaEventCreate(&e0));
	RT(cudaEventCreate(&e1));
	float ms;

	/* (1) populate on the host, then let GPU faults pull it in (the reference's fetch path) */
	double t0 = now_s();
	memset((void *)m, 3, bytes);
	double t_cpu = now_s() - t0;
	RT(cudaEventRecord(e0));
	touch_sum<<<g_sms * 8, 256>>>((const uint64_t *)m, bytes / 8, out);
	RT(cudaEventRecord(e1));
	RT(cudaEventSynchronize(e1));
	RT(cudaEventElapsedTime(&ms, e0, e1));
	printf("PROBE {\"section\":\"E\",\"what\":\"uvm_fault_h2d\",\"bytes\":%zu,\"ms\":%.2f,\"GBps\":%.2f,"
	       "\"cpu_first_touch_GBps\":%.2f}\n", bytes, ms, bytes / 1e9 / (ms * 1e-3), bytes / 1e9 / t_cpu);
	fflush(stdout);
	/* resident re-run */
	RT(cudaEventRecord(e0));
	touch_sum<<<g_sms * 8, 256>>>((const uint64_t *)m, bytes / 8, out);
	RT(cudaEventRecord(e1));
	RT(cudaEventSynchronize(e1));
	RT(cudaEventElapsedTime(&ms, e0, e1));
	printf("PROBE {\"section\":\"E\",\"what\":\"uvm_resident_read\",\"ms\":%.2f,\"GBps\":%.2f}\n", ms,
	       bytes / 1e9 / (ms * 1e-3));
	/* (2) prefetch-driven eviction and fetch */
	t0 = now_s();
	CU(cuMemPrefetchAsync(m, bytes, CU_DEVICE_CPU, 0));
	RT(cudaDeviceSynchronize());
	double t_out = now_s() - t0;
	t0 = now_s();
	CU(cuMemPrefetchAsync(m, bytes, g_dev, 0));
	RT(cudaDeviceSynchronize());
	double t_in = now_s() - t0;
	printf("PROBE {\"section\":\"E\",\"what\":\"uvm_prefetch\",\"d2h_GBps\":%.2f,\"h2d_GBps\":%.2f}\n",
	       bytes / 1e9 / t_out, bytes / 1e9 / t_in);
	/* (3) CPU faults pulling it back out (host read of device-resident managed memory) */
	t0 = now_s();
	volatile uint64_t acc = 0;
	for (size_t i = 0; i < bytes / 8; i += 512)
		acc += ((uint64_t *)m)[i];
	double t_cpuf = now_s() - t0;
	printf("PROBE {\"section\":\"E\",\"what\":\"uvm_cpu_fault_d2h\",\"GBps\":%.2f}\n", bytes / 1e9 / t_cpuf);
	fflush(stdout);
	CU(cuMemFree(m));
	cudaFree(out);
	return 0;
}

/* --------------------------------------------------------------- F ------ */
static int section_f(void)
{
	int ndev = 0;
	CU(cuDeviceGetCount(&ndev));
	if (ndev < 2) {
		printf("PROBE {\"section\":\"F\",\"skipped\":\"single device\"}\n");
		return 0;
	}
	const int peer = (g_dev + 1) % ndev;
	int can = 0;
	CU(cuDeviceCanAccessPeer(&can, g_dev, peer));
	printf("PROBE {\"section\":\"F\",\"peer\":%d,\"can_access\":%d}\n", peer, can);
	if (!can)
		return 0;
	/* physical memory on the peer, mapped read/write for the local device: no
	 * peer context, no cuCtxEnablePeerAccess -- exactly what the engine does */
	Bufs b;
	memset(&b, 0, sizeof b);
	b.bytes = g_scale_gib * GiB / 2;
	b.n_slabs = b.bytes / NVS_SLAB_BYTES;
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof prop);
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = peer;
	CUmemGenericAllocationHandle h;
	CU(cuMemCreate(&h, b.bytes, &prop, 0));
	CUdeviceptr pva = 0;
	CU(cuMemAddressReserve(&pva, b.bytes, 0, 0, 0));
	CU(cuMemMap(pva, b.bytes, 0, h, 0));
	CUmemAccessDesc acc[2];
	memset(acc, 0, sizeof acc);
	acc[0].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	acc[0].location.id = g_dev;
	acc[0].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	acc[1].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	acc[1].location.id = peer;
	acc[1].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	CU(cuMemSetAccess(pva, b.bytes, acc, 2));

	CU(cuMemAlloc(&b.dev_a, b.bytes));
	b.dev_b = pva; /* "d2d" now means local HBM -> peer HBM */
	CU(cuMemHostAlloc((void **)&b.descs_h, 2 * b.n_slabs * sizeof(nvs_copy_desc), CU_MEMHOSTALLOC_PORTABLE));
	RT(cudaMalloc(&b.descs_d[0], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.descs_d[1], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.counters, 64));
	RT(cudaMalloc(&b.mism, 8));
	for (int i = 0; i < 2; ++i)
		RT(cudaStreamCreateWithFlags(&b.st[i], cudaStreamNonBlocking));
	for (int i = 0; i < 4; ++i)
		RT(cudaEventCreate(&b.ev[i]));
	RT(cudaFuncSetAttribute(nvs_slab_copy_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
	if (fill(b, b.dev_a, 1))
		return -1;
	const int grids[] = {8, 16, 32, 66, 132};
	for (int pass = 0; pass < 2; ++pass) {
		/* pass 0: local -> peer (evict); pass 1: peer -> local (fetch) */
		if (pass == 1) {
			CUdeviceptr t = b.dev_a;
			b.dev_a = b.dev_b;
			b.dev_b = t;
		}
		Geo ce = {NVS_COPY_CE, 0, 0, 0, 0};
		printf("PROBE {\"section\":\"F\",\"pass\":\"%s\"}\n", pass ? "peer_to_local" : "local_to_peer");
		if (run_case(b, "d2d", ce, false, true)) return -1;
		for (int grid : grids) {
			Geo t = {NVS_COPY_TMA, grid, 1, 6, 32768};
			if (run_case(b, "d2d", t, false, grid == 132)) return -1;
			Geo t2 = {NVS_COPY_TMA, grid, 4, 3, 16384};
			if (run_case(b, "d2d", t2, false, grid == 132)) return -1;
			Geo l = {NVS_COPY_LDG, grid, 8, 0, 0};
			if (run_case(b, "d2d", l, false, grid == 132)) return -1;
		}
	}
	return 0;
}

/* --------------------------------------------------------------- G ------ */
/* Two PROCESSES sharing the GPU, one evicting (HBM->host) and one fetching
 * (host->HBM) at the same time: does the link run full duplex across contexts,
 * and does it depend on kernel vs copy engine?  (The engine's early-release
 * overlap is exactly this situation.) */
#include <sys/wait.h>
struct SharedG {
	volatile int ready;
	volatile int go;
	double gbps[2];
	double secs[2];
};

static int child_g(int role, int variant, SharedG *sh, int n_procs)
{
	if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
		return 1;
	CUdevice dev;
	cuDeviceGet(&dev, 0);
	cuDeviceGetAttribute(&g_sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev);
	Bufs b;
	memset(&b, 0, sizeof b);
	b.bytes = 4 * GiB;
	b.n_slabs = b.bytes / NVS_SLAB_BYTES;
	CU(cuMemAlloc(&b.dev_a, b.bytes));
	CU(cuMemHostAlloc((void **)&b.host_a, b.bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	CU(cuMemHostAlloc((void **)&b.descs_h, 2 * b.n_slabs * sizeof(nvs_copy_desc), CU_MEMHOSTALLOC_PORTABLE));
	RT(cudaMalloc(&b.descs_d[0], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.counters, 64));
	RT(cudaStreamCreateWithFlags(&b.st[0], cudaStreamNonBlocking));
	RT(cudaFuncSetAttribute(nvs_slab_copy_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
	memset(b.host_a, 1, b.bytes);
	RT(cudaMemset((void *)b.dev_a, 2, b.bytes));
	uint64_t src = role == 0 ? b.dev_a : (uint64_t)b.host_a;
	uint64_t dst = role == 0 ? (uint64_t)b.host_a : b.dev_a;
	build_descs(b, 0, src, dst);
	Geo g = {variant, 8, variant == NVS_COPY_LDG ? 8 : 1, 6, 32768};
	/* warm-up */
	if (variant == NVS_COPY_CE) {
		for (size_t off = 0; off < b.bytes; off += 64 * MiB)
			CU(cuMemcpyAsync(dst + off, src + off, 64 * MiB, b.st[0]));
	} else if (launch_copy(b, 0, g, b.st[0]))
		return 1;
	RT(cudaStreamSynchronize(b.st[0]));
	__sync_fetch_and_add(&sh->ready, 1);
	while (sh->ready < n_procs || !sh->go)
		usleep(100);
	const int reps = 6;
	double t0 = now_s();
	for (int r = 0; r < reps; ++r) {
		if (variant == NVS_COPY_CE) {
			for (size_t off = 0; off < b.bytes; off += 64 * MiB)
				CU(cuMemcpyAsync(dst + off, src + off, 64 * MiB, b.st[0]));
		} else if (launch_copy(b, 0, g, b.st[0]))
			return 1;
	}
	RT(cudaStreamSynchronize(b.st[0]));
	double t = now_s() - t0;
	sh->gbps[role] = reps * (double)b.bytes / 1e9 / t;
	sh->secs[role] = t;
	return 0;
}

static int section_g(void)
{
	SharedG *sh = (SharedG *)mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
	const int combos[][2] = {{NVS_COPY_TMA, -1}, {-1, NVS_COPY_TMA}, {NVS_COPY_CE, -1}, {-1, NVS_COPY_CE},
				 {NVS_COPY_TMA, NVS_COPY_TMA}, {NVS_COPY_CE, NVS_COPY_CE},
				 {NVS_COPY_TMA, NVS_COPY_CE}, {NVS_COPY_CE, NVS_COPY_TMA},
				 {NVS_COPY_LDG, NVS_COPY_LDG}};
	for (auto &c : combos) {
		memset((void *)sh, 0, sizeof *sh);
		int n_procs = (c[0] >= 0) + (c[1] >= 0);
		pid_t pids[2] = {0, 0};
		for (int role = 0; role < 2; ++role) {
			if (c[role] < 0)
				continue;
			pids[role] = fork();
			if (pids[role] == 0)
				_exit(child_g(role, c[role], sh, n_procs));
		}
		while (sh->ready < n_procs) {
			int st;
			pid_t w = waitpid(-1, &st, WNOHANG);
			if (w > 0) { printf("PROBE {\"section\":\"G\",\"error\":\"child died early\"}\n"); break; }
			usleep(1000);
		}
		sh->go = 1;
		for (int role = 0; role < 2; ++role)
			if (pids[role] > 0) {
				int st;
				waitpid(pids[role], &st, 0);
			}
		printf("PROBE {\"section\":\"G\",\"evict_variant\":\"%s\",\"fetch_variant\":\"%s\",\"evict_GBps\":%.2f,"
		       "\"fetch_GBps\":%.2f,\"sum_GBps\":%.2f,\"evict_s\":%.2f,\"fetch_s\":%.2f}\n",
		       c[0] < 0 ? "-" : vname(c[0]), c[1] < 0 ? "-" : vname(c[1]), sh->gbps[0], sh->gbps[1],
		       sh->gbps[0] + sh->gbps[1], sh->secs[0], sh->secs[1]);
		fflush(stdout);
	}
	return 0;
}

/* --------------------------------------------------------------- H ------ */
static long long read_ll(const char *path)
{
	FILE *f = fopen(path, "r");
	long long v = -1;
	if (f) {
		if (fscanf(f, "%lld", &v) != 1)
			v = -1;
		fclose(f);
	}
	return v;
}

static void *pin_worker(void *arg)
{
	CUcontext ctx = (CUcontext)arg;
	cuCtxSetCurrent(ctx);
	void *p = NULL;
	cuMemHostAlloc(&p, 2 * GiB, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP);
	return p;
}

static int section_h(void)
{
	const char *cur = "/sys/fs/cgroup/memory.current";
	long long limit = read_ll("/sys/fs/cgroup/memory.max");
	long long before = read_ll(cur);
	void *p = NULL;
	CU(cuMemHostAlloc(&p, 8 * GiB, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	memset(p, 1, 8 * GiB);
	long long after = read_ll(cur);
	printf("PROBE {\"section\":\"H\",\"what\":\"cuMemHostAlloc 8 GiB vs cgroup\",\"cgroup_limit\":%lld,"
	       "\"current_before\":%lld,\"current_after\":%lld,\"charged_bytes\":%lld}\n", limit, before, after, after - before);
	CU(cuMemFreeHost(p));
	/* UVM: host copies of evicted managed pages -- are THEY charged? */
	CUdeviceptr m = 0;
	CU(cuMemAllocManaged(&m, 8 * GiB, CU_MEM_ATTACH_GLOBAL));
	RT(cudaMemset((void *)m, 1, 8 * GiB));
	RT(cudaDeviceSynchronize());
	before = read_ll(cur);
	CU(cuMemPrefetchAsync(m, 8 * GiB, CU_DEVICE_CPU, 0));
	RT(cudaDeviceSynchronize());
	after = read_ll(cur);
	printf("PROBE {\"section\":\"H\",\"what\":\"8 GiB managed memory evicted to host vs cgroup\",\"charged_bytes\":%lld}\n",
	       after - before);
	CU(cuMemFree(m));
	/* does pinning parallelise across threads? */
	CUcontext ctx;
	CU(cuCtxGetCurrent(&ctx));
	for (int nt : {1, 4, 8}) {
		pthread_t th[8];
		double t0 = now_s();
		for (int i = 0; i < nt; ++i)
			pthread_create(&th[i], NULL, pin_worker, ctx);
		void *ptrs[8];
		for (int i = 0; i < nt; ++i)
			pthread_join(th[i], &ptrs[i]);
		double t = now_s() - t0;
		printf("PROBE {\"section\":\"H\",\"what\":\"parallel cuMemHostAlloc\",\"threads\":%d,\"GiB\":%d,\"seconds\":%.2f,"
		       "\"GBps\":%.2f}\n", nt, 2 * nt, t, 2.0 * nt * GiB / 1e9 / t);
		fflush(stdout);
		for (int i = 0; i < nt; ++i)
			if (ptrs[i])
				cuMemFreeHost(ptrs[i]);
	}
	return 0;
}

/* --------------------------------------------------------------- J ------ */
/* Why can cuMemUnmap + cuMemRelease cost far more per 256 MiB chunk inside a real
 * hand-off than section B measures?  Time them separately:
 * idle, beside our own copy kernel, beside another process's copy-engine traffic,
 * and with one cuMemUnmap spanning several chunks. */
struct JState {
	CUdeviceptr va;
	size_t chunk, n;
	std::vector<CUmemGenericAllocationHandle> h;
	CUmemAllocationProp prop;
	CUmemAccessDesc acc;
};

static int j_map_all(JState &j)
{
	for (size_t i = 0; i < j.n; ++i) {
		CU(cuMemCreate(&j.h[i], j.chunk, &j.prop, 0));
		CU(cuMemMap(j.va + i * j.chunk, j.chunk, 0, j.h[i], 0));
		CU(cuMemSetAccess(j.va + i * j.chunk, j.chunk, &j.acc, 1));
	}
	nvs_slab_fill<<<g_sms * 8, 256>>>((uint64_t *)j.va, j.n * j.chunk / 8, 0, 5);
	RT(cudaDeviceSynchronize());
	return 0;
}

static int j_unmap_all(JState &j, const char *label, size_t span)
{
	double t_unmap = 0, t_rel = 0, worst = 0;
	for (size_t i = 0; i < j.n; i += span) {
		double t0 = now_s();
		CU(cuMemUnmap(j.va + i * j.chunk, j.chunk * span));
		double t1 = now_s();
		for (size_t k = 0; k < span; ++k)
			CU(cuMemRelease(j.h[i + k]));
		double t2 = now_s();
		t_unmap += t1 - t0;
		t_rel += t2 - t1;
		if (t2 - t0 > worst)
			worst = t2 - t0;
	}
	printf("PROBE {\"section\":\"J\",\"case\":\"%s\",\"chunk_mib\":%zu,\"chunks\":%zu,\"span\":%zu,"
	       "\"unmap_ms_per_chunk\":%.3f,\"release_ms_per_chunk\":%.3f,\"worst_ms\":%.2f,\"GBps\":%.1f}\n",
	       label, j.chunk / MiB, j.n, span, t_unmap * 1e3 / j.n, t_rel * 1e3 / j.n, worst * 1e3,
	       j.n * j.chunk / 1e9 / (t_unmap + t_rel));
	fflush(stdout);
	return 0;
}

static int section_j(SharedG *sh)
{
	JState j;
	j.chunk = 256 * MiB;
	j.n = 64; /* 16 GiB */
	j.h.resize(j.n);
	memset(&j.prop, 0, sizeof j.prop);
	j.prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	j.prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	j.prop.location.id = g_dev;
	memset(&j.acc, 0, sizeof j.acc);
	j.acc.location = j.prop.location;
	j.acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	CU(cuMemAddressReserve(&j.va, j.n * j.chunk, 0, 0, 0));

	/* side traffic of our own: TMA D2H of a separate 2 GiB buffer, in a loop */
	Bufs b;
	memset(&b, 0, sizeof b);
	b.bytes = 2 * GiB;
	b.n_slabs = b.bytes / NVS_SLAB_BYTES;
	CU(cuMemAlloc(&b.dev_a, b.bytes));
	CU(cuMemHostAlloc((void **)&b.host_a, b.bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	CU(cuMemHostAlloc((void **)&b.descs_h, 2 * b.n_slabs * sizeof(nvs_copy_desc), CU_MEMHOSTALLOC_PORTABLE));
	RT(cudaMalloc(&b.descs_d[0], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.counters, 64));
	RT(cudaStreamCreateWithFlags(&b.st[0], cudaStreamNonBlocking));
	RT(cudaFuncSetAttribute(nvs_slab_copy_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
	build_descs(b, 0, b.dev_a, (uint64_t)b.host_a);
	Geo g = {NVS_COPY_TMA, 8, 1, 6, 32768};

	if (j_map_all(j)) return -1;
	if (j_unmap_all(j, "idle", 1)) return -1;

	if (j_map_all(j)) return -1;
	for (int r = 0; r < 24; ++r) /* ~1 s of queued copies */
		if (launch_copy(b, 0, g, b.st[0])) return -1;
	if (j_unmap_all(j, "beside own TMA copy kernel", 1)) return -1;
	RT(cudaDeviceSynchronize());

	if (j_map_all(j)) return -1;
	if (j_unmap_all(j, "idle, one unmap per 4 chunks", 4)) return -1;

	if (j_map_all(j)) return -1;
	for (int r = 0; r < 24; ++r)
		if (launch_copy(b, 0, g, b.st[0])) return -1;
	if (j_unmap_all(j, "beside own TMA copy kernel, one unmap per 4 chunks", 4)) return -1;
	RT(cudaDeviceSynchronize());

	/* cuMemGetInfo latency */
	{
		size_t f, t;
		double t0 = now_s();
		for (int i = 0; i < 2000; ++i)
			cuMemGetInfo(&f, &t);
		printf("PROBE {\"section\":\"J\",\"case\":\"cuMemGetInfo\",\"us_per_call\":%.2f}\n", (now_s() - t0) * 1e6 / 2000);
	}
	if (sh) {
		/* another process doing what a fetching client does */
		if (j_map_all(j)) return -1;
		sh->go = 1;
		usleep(300000);
		if (j_unmap_all(j, "beside another process (CE H2D + map churn)", 1)) return -1;
		if (j_map_all(j)) return -1;
		if (j_unmap_all(j, "beside another process, one unmap per 4 chunks", 4)) return -1;
		if (j_map_all(j)) return -1;
		for (int r = 0; r < 24; ++r)
			if (launch_copy(b, 0, g, b.st[0])) return -1;
		if (j_unmap_all(j, "beside another process AND own TMA kernel", 1)) return -1;
		RT(cudaDeviceSynchronize());
		sh->ready = 99; /* tell the child to stop */
	}
	return 0;
}

/* the "fetching client": copy-engine H2D in 256 MiB calls, plus create/map/release churn and cuMemGetInfo polling */
static int child_j(SharedG *sh)
{
	if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
		return 1;
	const size_t bytes = 4 * GiB, chunk = 256 * MiB;
	CUdeviceptr dev;
	uint8_t *host;
	CU(cuMemAlloc(&dev, bytes));
	CU(cuMemHostAlloc((void **)&host, bytes, CU_MEMHOSTALLOC_PORTABLE | CU_MEMHOSTALLOC_DEVICEMAP));
	memset(host, 1, bytes);
	cudaStream_t st;
	RT(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof prop);
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = 0;
	CUmemAccessDesc acc;
	memset(&acc, 0, sizeof acc);
	acc.location = prop.location;
	acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	CUdeviceptr va;
	CU(cuMemAddressReserve(&va, 8 * chunk, 0, 0, 0));
	while (!sh->go)
		usleep(100);
	unsigned long loops = 0;
	while (sh->ready != 99) {
		for (size_t off = 0; off < bytes; off += chunk)
			CU(cuMemcpyAsync(dev + off, (CUdeviceptr)host + off, chunk, st));
		for (int k = 0; k < 8; ++k) {
			CUmemGenericAllocationHandle h;
			size_t f, t;
			cuMemGetInfo(&f, &t);
			if (cuMemCreate(&h, chunk, &prop, 0) != CUDA_SUCCESS)
				continue;
			cuMemMap(va + k * chunk, chunk, 0, h, 0);
			cuMemSetAccess(va + k * chunk, chunk, &acc, 1);
			cuMemUnmap(va + k * chunk, chunk);
			cuMemRelease(h);
		}
		RT(cudaStreamSynchronize(st));
		++loops;
	}
	printf("PROBE {\"section\":\"J\",\"child_loops\":%lu}\n", loops);
	return 0;
}

static int section_j_two_process(void)
{
	SharedG *sh = (SharedG *)mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
	memset((void *)sh, 0, sizeof *sh);
	pid_t c = fork();
	if (c == 0)
		_exit(child_j(sh));
	if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
		return 1;
	CUdevice dev0;
	cuDeviceGet(&dev0, 0);
	cuDeviceGetAttribute(&g_sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev0);
	int rc = section_j(sh);
	sh->go = 1;
	sh->ready = 99;
	int st;
	waitpid(c, &st, 0);
	return rc;
}

/* --------------------------------------------------------------- K ------ */
/* The hand-off with HBM FULL: process A owns ~all free HBM in 256 MiB chunks and
 * gives it back chunk by chunk (unmap + release); process B grabs whatever
 * becomes free (create + map + setaccess), exactly like evict vs fetch but with
 * no data movement: a real hand-off can see per-chunk costs far above those of
 * section J (where HBM is never short).  Variants:
 *   mode 0  B polls cuMemGetInfo every 1 ms and maps as soon as one chunk fits
 *   mode 1  B maps only when >= 8 GiB are free (A runs ahead, calls interleave less)
 *   mode 2  B does not run at all (A alone, memory full at start)            */
struct SharedK {
	volatile int ready, go, done_a;
	volatile long b_chunks;
	double b_map_ms;
};

static int child_k(SharedK *sh, int mode, size_t chunk, size_t want_chunks)
{
	if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
		return 1;
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof prop);
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = 0;
	CUmemAccessDesc acc;
	memset(&acc, 0, sizeof acc);
	acc.location = prop.location;
	acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	CUdeviceptr va;
	CU(cuMemAddressReserve(&va, want_chunks * chunk, 0, 0, 0));
	std::vector<CUmemGenericAllocationHandle> h(want_chunks);
	__sync_fetch_and_add(&sh->ready, 1);
	while (!sh->go)
		usleep(100);
	size_t got = 0;
	double t_map = 0;
	const size_t need_free = mode == 1 ? 8 * GiB : chunk + 64 * MiB;
	while (got < want_chunks && !(sh->done_a && got >= want_chunks)) {
		size_t f = 0, t = 0;
		cuMemGetInfo(&f, &t);
		if (f < need_free && !(sh->done_a)) {
			usleep(1000);
			continue;
		}
		size_t burst = mode == 1 ? (f - 64 * MiB) / chunk : 1;
		for (size_t k = 0; k < burst && got < want_chunks; ++k) {
			double t0 = now_s();
			if (cuMemCreate(&h[got], chunk, &prop, 0) != CUDA_SUCCESS)
				break;
			cuMemMap(va + got * chunk, chunk, 0, h[got], 0);
			cuMemSetAccess(va + got * chunk, chunk, &acc, 1);
			t_map += now_s() - t0;
			++got;
			sh->b_chunks = (long)got;
		}
		if (sh->done_a && f < chunk + 64 * MiB)
			break;
	}
	sh->b_map_ms = t_map * 1e3;
	return 0;
}

static int section_k(void)
{
	const size_t chunk = 256 * MiB;
	for (int mode = 0; mode < 3; ++mode) {
		SharedK *sh = (SharedK *)mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
		memset((void *)sh, 0, sizeof *sh);
		const size_t n_give = 200; /* 50 GiB change hands */
		pid_t c = 0;
		if (mode != 2) {
			c = fork();
			if (c == 0)
				_exit(child_k(sh, mode, chunk, n_give));
		}
		pid_t a = fork();
		if (a == 0) {
			/* process A */
			if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
				_exit(1);
			CUdevice dev0;
			cuDeviceGet(&dev0, 0);
			cuDeviceGetAttribute(&g_sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev0);
			JState j;
			size_t f = 0, t = 0;
			cuMemGetInfo(&f, &t);
			j.chunk = chunk;
			j.n = (f - 1 * GiB) / chunk; /* take everything but ~1 GiB: HBM is now full */
			j.h.resize(j.n);
			memset(&j.prop, 0, sizeof j.prop);
			j.prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
			j.prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
			j.prop.location.id = 0;
			memset(&j.acc, 0, sizeof j.acc);
			j.acc.location = j.prop.location;
			j.acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
			if (cuMemAddressReserve(&j.va, j.n * j.chunk, 0, 0, 0) != CUDA_SUCCESS || j_map_all(j))
				_exit(2);
			while (mode != 2 && sh->ready < 1)
				usleep(100);
			sh->go = 1;
			usleep(50000);
			double t_unmap = 0, t_rel = 0, t0all = now_s();
			for (size_t i = 0; i < n_give; ++i) {
				double t0 = now_s();
				cuMemUnmap(j.va + i * j.chunk, j.chunk);
				double t1 = now_s();
				cuMemRelease(j.h[i]);
				t_unmap += t1 - t0;
				t_rel += now_s() - t1;
			}
			double wall = now_s() - t0all;
			sh->done_a = 1;
			printf("PROBE {\"section\":\"K\",\"mode\":%d,\"hbm_chunks_held\":%zu,\"given\":%zu,\"unmap_ms_per_chunk\":%.3f,"
			       "\"release_ms_per_chunk\":%.3f,\"wall_s\":%.3f,\"GBps\":%.1f}\n", mode, j.n, n_give,
			       t_unmap * 1e3 / n_give, t_rel * 1e3 / n_give, wall, n_give * chunk / 1e9 / wall);
			fflush(stdout);
			usleep(300000);
			_exit(0);
		}
		int st;
		waitpid(a, &st, 0);
		sh->done_a = 1;
		sh->go = 1;
		if (c > 0)
			waitpid(c, &st, 0);
		printf("PROBE {\"section\":\"K\",\"mode\":%d,\"b_chunks\":%ld,\"b_map_ms_per_chunk\":%.3f}\n", mode, sh->b_chunks,
		       sh->b_chunks ? sh->b_map_ms / sh->b_chunks : 0.0);
		fflush(stdout);
	}
	return 0;
}

/* --------------------------------------------------------------- L ------ */
/* Handing PHYSICAL chunks over instead of release -> poll -> create (VERDICT r1 #4): A owns ~all
 * of the HBM in 256 MiB chunks created with a POSIX-fd shareable handle type; for each chunk it
 * exports the handle, sends the fd over a Unix socket (SCM_RIGHTS), unmaps and releases; B imports,
 * maps and sets access.  No cuMemCreate / cuMemGetInfo polling on B's side, the memory never
 * becomes "free" in between.  Also: does asking for a shareable handle type make cuMemCreate slower? */
#include <sys/socket.h>
#include <sys/wait.h>
static int send_fd(int sock, int fd)
{
	char byte = 'F', ctrl[CMSG_SPACE(sizeof(int))];
	struct iovec io = {&byte, 1};
	struct msghdr m;
	memset(&m, 0, sizeof m);
	memset(ctrl, 0, sizeof ctrl);
	m.msg_iov = &io;
	m.msg_iovlen = 1;
	m.msg_control = ctrl;
	m.msg_controllen = sizeof ctrl;
	struct cmsghdr *c = CMSG_FIRSTHDR(&m);
	c->cmsg_level = SOL_SOCKET;
	c->cmsg_type = SCM_RIGHTS;
	c->cmsg_len = CMSG_LEN(sizeof(int));
	memcpy(CMSG_DATA(c), &fd, sizeof(int));
	return sendmsg(sock, &m, 0) == 1 ? 0 : -1;
}

static int recv_fd(int sock)
{
	char byte, ctrl[CMSG_SPACE(sizeof(int))];
	struct iovec io = {&byte, 1};
	struct msghdr m;
	memset(&m, 0, sizeof m);
	m.msg_iov = &io;
	m.msg_iovlen = 1;
	m.msg_control = ctrl;
	m.msg_controllen = sizeof ctrl;
	if (recvmsg(sock, &m, 0) != 1)
		return -1;
	struct cmsghdr *c = CMSG_FIRSTHDR(&m);
	int fd = -1;
	if (c && c->cmsg_type == SCM_RIGHTS)
		memcpy(&fd, CMSG_DATA(c), sizeof(int));
	return fd;
}

static int section_l(void)
{
	const size_t chunk = 256 * MiB, n_give = 200;
	int sv[2];
	if (socketpair(AF_UNIX, SOCK_STREAM, 0, sv) != 0)
		return -1;
	SharedK *sh = (SharedK *)mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
	memset((void *)sh, 0, sizeof *sh);
	pid_t b = fork();
	if (b == 0) { /* process B: imports what A hands over */
		close(sv[0]);
		if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
			_exit(1);
		CUmemAccessDesc acc;
		memset(&acc, 0, sizeof acc);
		acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
		acc.location.id = 0;
		acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
		CUdeviceptr va;
		if (cuMemAddressReserve(&va, n_give * chunk, 0, 0, 0) != CUDA_SUCCESS)
			_exit(2);
		std::vector<CUmemGenericAllocationHandle> h(n_give);
		__sync_fetch_and_add(&sh->ready, 1);
		double t_imp = 0, t_map = 0, t_acc = 0, t_recv = 0;
		size_t got = 0;
		unsigned long long first_word = 0;
		for (; got < n_give; ++got) {
			double t0 = now_s();
			int fd = recv_fd(sv[1]);
			if (fd < 0)
				break;
			double t1 = now_s();
			if (cuMemImportFromShareableHandle(&h[got], (void *)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) != CUDA_SUCCESS)
				break;
			double t2 = now_s();
			cuMemMap(va + got * chunk, chunk, 0, h[got], 0);
			double t3 = now_s();
			cuMemSetAccess(va + got * chunk, chunk, &acc, 1);
			double t4 = now_s();
			close(fd);
			t_recv += t1 - t0;
			t_imp += t2 - t1;
			t_map += t3 - t2;
			t_acc += t4 - t3;
			if (got == 0)
				cudaMemcpy(&first_word, (void *)va, 8, cudaMemcpyDeviceToHost);
		}
		printf("PROBE {\"section\":\"L\",\"side\":\"B\",\"chunks\":%zu,\"recv_wait_ms_per_chunk\":%.3f,\"import_ms_per_chunk\":%.3f,"
		       "\"map_ms_per_chunk\":%.3f,\"setaccess_ms_per_chunk\":%.3f,\"first_word\":\"%llx\"}\n", got,
		       t_recv * 1e3 / n_give, t_imp * 1e3 / n_give, t_map * 1e3 / n_give, t_acc * 1e3 / n_give, first_word);
		fflush(stdout);
		_exit(got == n_give ? 0 : 3);
	}
	pid_t a = fork();
	if (a == 0) { /* process A: owns the HBM, hands n_give chunks over */
		close(sv[1]);
		if (cuInit(0) != CUDA_SUCCESS || cudaSetDevice(0) != cudaSuccess || cudaFree(0) != cudaSuccess)
			_exit(1);
		JState j;
		size_t f = 0, t = 0;
		cuMemGetInfo(&f, &t);
		j.chunk = chunk;
		j.n = (f - 1 * GiB) / chunk;
		j.h.resize(j.n);
		memset(&j.prop, 0, sizeof j.prop);
		j.prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
		j.prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
		j.prop.location.id = 0;
		j.prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
		memset(&j.acc, 0, sizeof j.acc);
		j.acc.location = j.prop.location;
		j.acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
		double t0 = now_s();
		if (cuMemAddressReserve(&j.va, j.n * j.chunk, 0, 0, 0) != CUDA_SUCCESS || j_map_all(j))
			_exit(2);
		double t_fill = now_s() - t0;
		unsigned long long magic = 0xfeedfacecafe1234ull;
		cudaMemcpy((void *)j.va, &magic, 8, cudaMemcpyHostToDevice);
		while (sh->ready < 1)
			usleep(100);
		double t_exp = 0, t_send = 0, t_unmap = 0, t_rel = 0, t0all = now_s();
		for (size_t i = 0; i < n_give; ++i) {
			int fd = -1;
			double a0 = now_s();
			if (cuMemExportToShareableHandle(&fd, j.h[i], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) != CUDA_SUCCESS)
				_exit(4);
			double a1 = now_s();
			send_fd(sv[0], fd);
			double a2 = now_s();
			cuMemUnmap(j.va + i * j.chunk, j.chunk);
			double a3 = now_s();
			cuMemRelease(j.h[i]);
			close(fd);
			double a4 = now_s();
			t_exp += a1 - a0;
			t_send += a2 - a1;
			t_unmap += a3 - a2;
			t_rel += a4 - a3;
		}
		double wall = now_s() - t0all;
		printf("PROBE {\"section\":\"L\",\"side\":\"A\",\"hbm_chunks_held\":%zu,\"create_map_ms_per_chunk_shareable\":%.3f,\"given\":%zu,"
		       "\"export_ms_per_chunk\":%.3f,\"send_ms_per_chunk\":%.3f,\"unmap_ms_per_chunk\":%.3f,\"release_ms_per_chunk\":%.3f,"
		       "\"wall_s\":%.3f,\"GBps\":%.1f}\n", j.n, t_fill * 1e3 / j.n, n_give, t_exp * 1e3 / n_give, t_send * 1e3 / n_give,
		       t_unmap * 1e3 / n_give, t_rel * 1e3 / n_give, wall, n_give * chunk / 1e9 / wall);
		fflush(stdout);
		usleep(500000);
		_exit(0);
	}
	close(sv[0]);
	close(sv[1]);
	int st;
	waitpid(a, &st, 0);
	waitpid(b, &st, 0);
	return 0;
}

/* --------------------------------------------------------------- I ------ */
/* The shared host pool: a /dev/shm file, pages faulted in by 8 threads (reads),
 * pinned with cuMemHostRegister.  How fast is provisioning, and is the link
 * bandwidth to such memory the same as to cuMemHostAlloc memory? */
#include <fcntl.h>
static void *touch_ro(void *arg)
{
	volatile const uint8_t *p = (volatile const uint8_t *)((void **)arg)[0];
	size_t n = (size_t)((void **)arg)[1];
	uint8_t acc = 0;
	for (size_t off = 0; off < n; off += 4096)
		acc ^= p[off];
	return (void *)(uintptr_t)acc;
}

static int section_i(void)
{
	const size_t bytes = 4 * GiB;
	const char *path = "/dev/shm/nvs_probe_pool";
	unlink(path);
	int fd = open(path, O_RDWR | O_CREAT, 0600);
	if (fd < 0 || ftruncate(fd, bytes) != 0) {
		printf("PROBE {\"section\":\"I\",\"error\":\"shm file\"}\n");
		return -1;
	}
	uint8_t *p = (uint8_t *)mmap(NULL, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
	if (p == MAP_FAILED)
		return -1;
	double t0 = now_s();
	enum { NTT = 32 };
	pthread_t th[NTT];
	void *args[NTT][2];
	for (int i = 0; i < NTT; ++i) {
		args[i][0] = p + bytes / NTT * i;
		args[i][1] = (void *)(bytes / NTT);
		pthread_create(&th[i], NULL, touch_ro, args[i]);
	}
	for (int i = 0; i < NTT; ++i)
		pthread_join(th[i], NULL);
	double t_touch = now_s() - t0;
	t0 = now_s();
	CUresult r = cuMemHostRegister(p, bytes, CU_MEMHOSTREGISTER_PORTABLE | CU_MEMHOSTREGISTER_DEVICEMAP);
	double t_reg = now_s() - t0;
	CUdeviceptr dp = 0;
	if (r == CUDA_SUCCESS)
		cuMemHostGetDevicePointer(&dp, p, 0);
	printf("PROBE {\"section\":\"I\",\"what\":\"shm pool provisioning\",\"bytes\":%zu,\"touch8_GBps\":%.2f,"
	       "\"register_rc\":%d,\"register_GBps\":%.2f,\"overall_GBps\":%.2f,\"dev_eq_host\":%d}\n",
	       bytes, bytes / 1e9 / t_touch, (int)r, bytes / 1e9 / t_reg, bytes / 1e9 / (t_touch + t_reg),
	       dp == (CUdeviceptr)(uintptr_t)p);
	fflush(stdout);
	if (r != CUDA_SUCCESS)
		return -1;
	/* second registration of pages that already exist (what the 2nd client does) */
	uint8_t *q = (uint8_t *)mmap(NULL, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
	t0 = now_s();
	r = cuMemHostRegister(q, bytes, CU_MEMHOSTREGISTER_PORTABLE | CU_MEMHOSTREGISTER_DEVICEMAP);
	printf("PROBE {\"section\":\"I\",\"what\":\"second mapping register\",\"rc\":%d,\"GBps\":%.2f}\n", (int)r,
	       bytes / 1e9 / (now_s() - t0));
	if (r == CUDA_SUCCESS)
		cuMemHostUnregister(q);
	munmap(q, bytes);

	Bufs b;
	memset(&b, 0, sizeof b);
	b.bytes = bytes;
	b.n_slabs = b.bytes / NVS_SLAB_BYTES;
	CU(cuMemAlloc(&b.dev_a, b.bytes));
	CU(cuMemAlloc(&b.dev_b, b.bytes));
	b.host_a = (uint8_t *)dp;
	b.host_b = (uint8_t *)dp;
	CU(cuMemHostAlloc((void **)&b.descs_h, 2 * b.n_slabs * sizeof(nvs_copy_desc), CU_MEMHOSTALLOC_PORTABLE));
	RT(cudaMalloc(&b.descs_d[0], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.descs_d[1], b.n_slabs * sizeof(nvs_copy_desc)));
	RT(cudaMalloc(&b.counters, 64));
	RT(cudaMalloc(&b.mism, 8));
	for (int i = 0; i < 2; ++i)
		RT(cudaStreamCreateWithFlags(&b.st[i], cudaStreamNonBlocking));
	for (int i = 0; i < 4; ++i)
		RT(cudaEventCreate(&b.ev[i]));
	RT(cudaFuncSetAttribute(nvs_slab_copy_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
	if (fill(b, b.dev_a, 1))
		return -1;
	Geo t = {NVS_COPY_TMA, 8, 1, 6, 32768};
	Geo ce = {NVS_COPY_CE, 0, 0, 0, 0};
	if (run_case(b, "d2h", t, false, true)) return -1;
	if (run_case(b, "h2d", t, false, true)) return -1;
	if (run_case(b, "d2h", ce, false, true)) return -1;
	if (run_case(b, "h2d", ce, false, true)) return -1;
	/* the CPU sees what the GPU wrote through the registration */
	unsigned long long bad = 0;
	for (size_t i = 0; i < bytes / 8; i += 4099)
		bad += ((uint64_t *)p)[i] != nvs_pattern(i, 1);
	printf("PROBE {\"section\":\"I\",\"what\":\"cpu view of shm after d2h\",\"sampled_mismatches\":%llu}\n", bad);
	cuMemHostUnregister(p);
	munmap(p, bytes);
	close(fd);
	unlink(path);
	cuMemFree(b.dev_a);
	cuMemFree(b.dev_b);
	return 0;
}

int main(int argc, char **argv)
{
	const char *sections = argc > 1 ? argv[1] : "ABCDEF";
	if (argc > 1 && !strcmp(argv[1], "G")) /* forks before any CUDA initialisation */
		return section_g();
	if (argc > 1 && !strcmp(argv[1], "J"))
		return section_j_two_process();
	if (argc > 1 && !strcmp(argv[1], "K"))
		return section_k();
	if (argc > 1 && !strcmp(argv[1], "L"))
		return section_l();
	if (argc > 2)
		g_scale_gib = strtoull(argv[2], NULL, 0);
	if (cuInit(0) != CUDA_SUCCESS) {
		printf("PROBE {\"error\":\"cuInit\"}\n");
		return 1;
	}
	if (cudaSetDevice(g_dev) != cudaSuccess || cudaFree(0) != cudaSuccess) {
		printf("PROBE {\"error\":\"cudaSetDevice\"}\n");
		return 1;
	}
	{
		CUdevice dev0;
		cuDeviceGet(&dev0, g_dev);
		cuDeviceGetAttribute(&g_sms, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev0);
	}
	int rc = 0;
	for (const char *s = sections; *s; ++s) {
		double t0 = now_s();
		int r = 0;
		switch (*s) {
		case 'A': r = section_a(); break;
		case 'B': r = section_b(); break;
		case 'C': r = section_c(); break;
		case 'D': r = section_d(); break;
		case 'E': r = section_e(); break;
		case 'F': r = section_f(); break;
		case 'H': r = section_h(); break;
		case 'I': r = section_i(); break;
		default: break;
		}
		printf("PROBE {\"section_done\":\"%c\",\"rc\":%d,\"seconds\":%.1f}\n", *s, r, now_s() - t0);
		fflush(stdout);
		if (r) {
			rc = 1;
			cudaDeviceSynchronize();
			cudaGetLastError();
		}
	}
	return rc;
}
