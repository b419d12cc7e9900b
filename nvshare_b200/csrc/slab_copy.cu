/*
 * slab_copy.cu -- the hot kernel of the H100 swap engine (sm_90a only).
 *
 * What it replaces: in the reference, the bytes of an oversubscribed
 * allocation move between HBM and host DRAM inside NVIDIA's UVM driver, one
 * GPU page fault batch at a time, after real_cuMemAllocManaged()
 * (reference src/hook.c:673) and the first touch following LOCK_OK
 * (reference src/client.c:298-307).  Here the move is explicit: the host engine
 * (engine.c) hands this kernel a list of nvs_copy_desc (<= 2 MiB each) and a
 * few resident CTAs stream them.
 *
 * Three entry points, all `extern "C"` so the engine can cuModuleGetFunction
 * them from the embedded cubin:
 *
 *   nvs_slab_copy_tma   one elected lane per warp drives a ring of S smem
 *                       stages with cp.async.bulk (TMA, non-tensor):
 *                         global --(bulk load, mbarrier complete_tx)--> smem
 *                         smem   --(bulk store, bulk_group)-----------> global
 *                       No register staging, no generic-proxy access to the
 *                       payload at all; S-1 loads are always in flight per warp.
 *   nvs_slab_copy_ldg   all lanes, 16-byte ld.global.cs / st.global.cs, 8 loads
 *                       in flight per thread before the first store.
 *   nvs_slab_verify     parity helper: counts 64-bit words that differ from the
 *                       position-dependent pattern (used by tests / bench; it
 *                       can read pinned host and peer memory as well).
 *   nvs_slab_fill       writes that pattern.
 *
 * Bound: link bandwidth (PCIe Gen5 x16 or NVLink 4), not HBM and not tensor
 * cores -- see DESIGN.md.  Work is distributed dynamically (one atomicAdd per
 * descriptor) so CTAs that share an SM with a client's kernels simply take
 * fewer slabs.
 */
#include <stdint.h>
#include "../../include/nvs_copy_desc.h"

#define NVS_MAX_WARPS  8
#define NVS_MAX_STAGES 8

/* ------------------------------------------------------------------ PTX -- */

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
	return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
		     : "memory");
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
	asm volatile(
		"{\n\t"
		".reg .pred p;\n\t"
		"NVS_WAIT_%=:\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
		"@p bra NVS_DONE_%=;\n\t"
		"bra NVS_WAIT_%=;\n\t"
		"NVS_DONE_%=:\n\t"
		"}\n" ::"r"(bar),
		"r"(parity)
		: "memory");
}

/* global -> shared::cta, completion counted in bytes on an mbarrier (SASS: UBLKCP) */
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, uint64_t src_gmem, uint32_t bytes,
					 uint32_t bar)
{
	asm volatile(
		"cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
		::"r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar)
		: "memory");
}

/* shared::cta -> global, tracked by the per-thread bulk async-group */
__device__ __forceinline__ void bulk_s2g(uint64_t dst_gmem, uint32_t src_smem, uint32_t bytes)
{
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem),
		     "r"(src_smem), "r"(bytes)
		     : "memory");
}

__device__ __forceinline__ void bulk_commit(void)
{
	asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

/* all but the most recent 1 group have finished READING their smem source */
__device__ __forceinline__ void bulk_wait_read_1(void)
{
	asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}

/* every group fully complete (writes performed) */
__device__ __forceinline__ void bulk_wait_all(void)
{
	asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

/* ------------------------------------------------- TMA (bulk) variant ---- */

/*
 * Launch: grid = any, block = 32 * n_warps (n_warps <= NVS_MAX_WARPS),
 * dynamic smem = n_warps * n_stages * tile_bytes (+ alignment slack of 128).
 * tile_bytes must be a multiple of 16; 2 <= n_stages <= NVS_MAX_STAGES.
 * `counter` points to one zeroed uint32 in device memory per launch.
 */
extern "C" __global__ void __launch_bounds__(32 * NVS_MAX_WARPS, 1)
nvs_slab_copy_tma(const nvs_copy_desc *__restrict__ descs, uint32_t n_descs, uint32_t *counter,
		  uint32_t tile_bytes, uint32_t n_stages)
{
	extern __shared__ __align__(128) uint8_t smem_raw[];
	__shared__ __align__(8) uint64_t full_bar[NVS_MAX_WARPS][NVS_MAX_STAGES];
	__shared__ uint64_t tile_dst[NVS_MAX_WARPS][NVS_MAX_STAGES];
	__shared__ uint32_t tile_len[NVS_MAX_WARPS][NVS_MAX_STAGES];

	const uint32_t warp = threadIdx.x >> 5;
	if ((threadIdx.x & 31u) != 0)
		return; /* one driving lane per warp; TMA does the moving */

	const uint32_t S = n_stages;
	const uint32_t T = tile_bytes;
	const uint32_t ring = smem_u32(smem_raw) + warp * S * T;

	for (uint32_t s = 0; s < S; ++s)
		mbar_init(smem_u32(&full_bar[warp][s]), 1);
	/* make the inits visible to the async proxy before the first bulk copy */
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

	uint64_t cur_src = 0, cur_dst = 0, rem = 0;
	uint32_t issued = 0, consumed = 0;
	bool drained = false; /* work queue exhausted */

	/* issue the load of the next tile of the descriptor stream; false when none left */
	auto produce = [&]() -> bool {
		while (rem == 0) {
			if (drained)
				return false;
			const uint32_t idx = atomicAdd(counter, 1u);
			if (idx >= n_descs) {
				drained = true;
				return false;
			}
			cur_src = descs[idx].src;
			cur_dst = descs[idx].dst;
			rem = descs[idx].bytes; /* 0-byte descriptors are skipped */
		}
		const uint32_t b = rem < (uint64_t)T ? (uint32_t)rem : T;
		const uint32_t s = issued % S;
		const uint32_t bar = smem_u32(&full_bar[warp][s]);
		tile_dst[warp][s] = cur_dst;
		tile_len[warp][s] = b;
		mbar_expect_tx(bar, b);
		bulk_g2s(ring + s * T, cur_src, b, bar);
		cur_src += b;
		cur_dst += b;
		rem -= b;
		++issued;
		return true;
	};

	/* prologue: S-1 loads in flight */
	for (uint32_t i = 0; i + 1 < S; ++i)
		if (!produce())
			break;

	while (consumed < issued) {
		const uint32_t s = consumed % S;
		mbar_wait(smem_u32(&full_bar[warp][s]), (consumed / S) & 1u);
		bulk_s2g(tile_dst[warp][s], ring + s * T, tile_len[warp][s]);
		bulk_commit();
		++consumed;
		/*
		 * Refill.  Lookahead is S-1, so the stage the next load lands in
		 * (issued % S) was last read by the store of tile consumed - 2:
		 * every bulk group except the one just committed must have finished
		 * reading shared memory.
		 */
		if (!(drained && rem == 0)) {
			bulk_wait_read_1();
			produce();
		}
	}
	bulk_wait_all();
}

/* ------------------------------------------------- LDG/STG variant ------- */

#define NVS_LDG_UNROLL 8

/*
 * Launch: grid = any, block = any multiple of 32 (256 recommended), no dynamic
 * smem.  One CTA takes one descriptor at a time.
 */
extern "C" __global__ void __launch_bounds__(1024)
nvs_slab_copy_ldg(const nvs_copy_desc *__restrict__ descs, uint32_t n_descs, uint32_t *counter)
{
	__shared__ uint32_t s_idx;
	for (;;) {
		__syncthreads();
		if (threadIdx.x == 0)
			s_idx = atomicAdd(counter, 1u);
		__syncthreads();
		const uint32_t idx = s_idx;
		if (idx >= n_descs)
			return;
		const int4 *__restrict__ src = reinterpret_cast<const int4 *>(descs[idx].src);
		int4 *__restrict__ dst = reinterpret_cast<int4 *>(descs[idx].dst);
		const uint64_t n16 = descs[idx].bytes >> 4;
		const uint64_t step = (uint64_t)blockDim.x * NVS_LDG_UNROLL;
		uint64_t base = 0;
		for (; base + step <= n16; base += step) {
			int4 v[NVS_LDG_UNROLL];
#pragma unroll
			for (int u = 0; u < NVS_LDG_UNROLL; ++u)
				v[u] = __ldcs(src + base + (uint64_t)u * blockDim.x + threadIdx.x);
#pragma unroll
			for (int u = 0; u < NVS_LDG_UNROLL; ++u)
				__stcs(dst + base + (uint64_t)u * blockDim.x + threadIdx.x, v[u]);
		}
		for (uint64_t i = base + threadIdx.x; i < n16; i += blockDim.x)
			__stcs(dst + i, __ldcs(src + i));
		/* sub-16-byte tail (never produced by the engine; kept for the C-ABI) */
		const uint64_t tail = descs[idx].bytes & 15ull;
		if (threadIdx.x < tail) {
			const uint8_t *s8 = reinterpret_cast<const uint8_t *>(descs[idx].src) + (n16 << 4);
			uint8_t *d8 = reinterpret_cast<uint8_t *>(descs[idx].dst) + (n16 << 4);
			d8[threadIdx.x] = s8[threadIdx.x];
		}
	}
}

/* --------------------------- same-filled slab elision + clean-slab hash ----- */

/*
 * Two ways of not moving a slab at all, both decided by ONE pass of the SMs over it
 * at HBM speed (tens of times the PCIe link, several times NVLink) -- the copy engines cannot do either:
 *
 *  - same-filled: all 64-bit words equal (zero-initialised buffers, ones(), padding,
 *    memset workspaces -- the reference's own test tensors are torch.ones): 8 bytes
 *    describe it, nvs_slab_splat re-creates it at fetch.
 *  - clean: the backing copy kept from the last hand-off still matches.  VMM memory
 *    has no dirty bits, so "matches" is decided by a 128-bit content hash of the slab
 *    compared with the hash recorded when that backing copy was written.
 *
 *   nvs_slab_scan    one CTA (256 threads) per slab: out[i] = {word 0, all words
 *                    equal?, h0, h1}.  want_hash == 0: leaves the slab at the first
 *                    32 KiB tile that differs (h0 = h1 = 0).  want_hash != 0: reads
 *                    every byte.  A descriptor with dst != 0 is a FUSED copy + hash:
 *                    every 16-byte vector a lane loads is hashed and stored to dst by
 *                    that same lane, so the hash describes exactly the bytes that
 *                    landed in dst even while other kernels are writing the source
 *                    (background pre-cleaning: the engine writes resident chunks back
 *                    during their owner's quantum, when the link is idle, and no
 *                    second pass over the copy is needed to know what it holds).
 *   nvs_slab_splat   the inverse of same-filled: fill dst with the 64-bit value
 *
 * The hash (restated in C by oracle/nvshare_oracle.c: oracle_slab_hash, and checked
 * against it bit for bit on the GPU).  The slab is a sequence of 16-byte vectors
 * (x, y, z, w); lane t of 256 owns vectors t, t+256, t+512, ... in that order and runs
 * four independent xxHash32 rounds over them,
 *      a_k = rotl32(a_k + word_k * P2, 13) * P1        a_k(0) = SEED_k ^ (t * P1)
 * each of which is a bijection of a_k for a fixed word and injective in the word for a
 * fixed a_k.  A lane's four accumulators go through a 128-bit bijection (two Feistel
 * steps + SplitMix64 finalisers, lane index mixed in) and the slab hash is the pair of
 * 64-bit sums over the lanes.  Consequences: ANY change confined to one lane's stream
 * (in particular any single-word change) is detected with certainty; changes spread
 * over several lanes escape with probability ~2^-128.  12 integer instructions per
 * 16 bytes: the pass stays HBM-bound (132 SMs x 128 lanes x 1.98 GHz / 12 x 16 B = 45 TB/s
 * of hashing capacity against the 3.35 TB/s of HBM3 the H100 SXM data sheet gives).
 */
struct nvs_scan_result {
	unsigned long long value;
	unsigned long long is_const;
	unsigned long long h0, h1;
};

#define NVS_SCAN_THREADS 256
#define NVS_SCAN_UNROLL 8
#define NVS_H_P1 0x9E3779B1u
#define NVS_H_P2 0x85EBCA77u

__host__ __device__ __forceinline__ uint32_t nvs_rotl32(uint32_t x, int r)
{
	return (x << r) | (x >> (32 - r));
}

__host__ __device__ __forceinline__ unsigned long long nvs_mix64(unsigned long long z)
{
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

#define NVS_H_ROUND(a, w) a = nvs_rotl32((a) + (w) * NVS_H_P2, 13) * NVS_H_P1

extern "C" __global__ void __launch_bounds__(NVS_SCAN_THREADS)
nvs_slab_scan(const nvs_copy_desc *__restrict__ descs, uint32_t n_descs, uint32_t *counter,
	      nvs_scan_result *__restrict__ out, uint32_t want_hash)
{
	__shared__ uint32_t s_idx;
	__shared__ unsigned long long s_red[2][NVS_SCAN_THREADS / 32];
	const uint32_t t = threadIdx.x;
	for (;;) {
		__syncthreads();
		if (t == 0)
			s_idx = atomicAdd(counter, 1u);
		__syncthreads();
		const uint32_t idx = s_idx;
		if (idx >= n_descs)
			return;
		const uint4 *__restrict__ p = reinterpret_cast<const uint4 *>(descs[idx].src);
		uint4 *__restrict__ q = reinterpret_cast<uint4 *>(descs[idx].dst); /* NULL: scan only */
		const uint64_t n16 = descs[idx].bytes >> 4;
		const unsigned long long v0 = reinterpret_cast<const unsigned long long *>(descs[idx].src)[0];
		const uint32_t v0lo = (uint32_t)v0, v0hi = (uint32_t)(v0 >> 32);
		const uint64_t step = (uint64_t)NVS_SCAN_THREADS * NVS_SCAN_UNROLL;
		uint32_t a0 = 0x243F6A88u ^ (t * NVS_H_P1), a1 = 0x85A308D3u ^ (t * NVS_H_P1);
		uint32_t a2 = 0x13198A2Eu ^ (t * NVS_H_P1), a3 = 0x03707344u ^ (t * NVS_H_P1);
		int differs = 0;
		for (uint64_t base = 0; base < n16; base += step) {
			uint4 v[NVS_SCAN_UNROLL];
			bool live[NVS_SCAN_UNROLL];
#pragma unroll
			for (int u = 0; u < NVS_SCAN_UNROLL; ++u) {
				const uint64_t i = base + (uint64_t)u * NVS_SCAN_THREADS + t;
				live[u] = i < n16;
				v[u] = live[u] ? __ldcs(p + i) : make_uint4(v0lo, v0hi, v0lo, v0hi);
			}
			int d = 0;
#pragma unroll
			for (int u = 0; u < NVS_SCAN_UNROLL; ++u) {
				d |= (v[u].x != v0lo) | (v[u].y != v0hi) | (v[u].z != v0lo) | (v[u].w != v0hi);
				if (live[u]) {
					if (q)
						__stcs(q + base + (uint64_t)u * NVS_SCAN_THREADS + t, v[u]);
					NVS_H_ROUND(a0, v[u].x);
					NVS_H_ROUND(a1, v[u].y);
					NVS_H_ROUND(a2, v[u].z);
					NVS_H_ROUND(a3, v[u].w);
				}
			}
			differs |= d;
			if (!want_hash && !q && __syncthreads_or(d)) {
				differs = 1;
				break;
			}
		}
		/* lane (a0..a3) -> 128 bits, bijectively, with the lane index mixed in */
		unsigned long long u64 = ((unsigned long long)a0 << 32) | a1, w64 = ((unsigned long long)a2 << 32) | a3;
		u64 ^= (unsigned long long)(t + 1) * 0x9E3779B97F4A7C15ull;
		w64 ^= nvs_mix64(u64);
		u64 ^= nvs_mix64(w64 + 0xD1B54A32D192ED03ull);
		unsigned long long h0 = nvs_mix64(u64), h1 = nvs_mix64(w64);
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			h0 += __shfl_xor_sync(0xffffffffu, h0, o);
			h1 += __shfl_xor_sync(0xffffffffu, h1, o);
		}
		if ((t & 31u) == 0) {
			s_red[0][t >> 5] = h0;
			s_red[1][t >> 5] = h1;
		}
		const int any_differs = __syncthreads_or(differs);
		if (t == 0) {
			unsigned long long s0 = 0, s1 = 0;
#pragma unroll
			for (int w = 0; w < NVS_SCAN_THREADS / 32; ++w) {
				s0 += s_red[0][w];
				s1 += s_red[1][w];
			}
			out[idx].value = v0;
			out[idx].is_const = !any_differs && (descs[idx].bytes & 15ull) == 0;
			out[idx].h0 = (want_hash || q) ? s0 : 0ull;
			out[idx].h1 = (want_hash || q) ? s1 : 0ull;
		}
	}
}

extern "C" __global__ void __launch_bounds__(256)
nvs_slab_splat(const nvs_copy_desc *__restrict__ descs, uint32_t n_descs, uint32_t *counter)
{
	__shared__ uint32_t s_idx;
	for (;;) {
		__syncthreads();
		if (threadIdx.x == 0)
			s_idx = atomicAdd(counter, 1u);
		__syncthreads();
		const uint32_t idx = s_idx;
		if (idx >= n_descs)
			return;
		const unsigned long long v = descs[idx].src; /* the value, not an address */
		ulonglong2 *__restrict__ q = reinterpret_cast<ulonglong2 *>(descs[idx].dst);
		const uint64_t n16 = descs[idx].bytes >> 4;
		const ulonglong2 vv = make_ulonglong2(v, v);
		for (uint64_t i = threadIdx.x; i < n16; i += blockDim.x)
			__stcs(q + i, vv);
	}
}

/* ------------------------------------------------- pattern helpers ------- */

/* position-dependent 64-bit pattern: distinguishes every word of every slab */
__host__ __device__ __forceinline__ uint64_t nvs_pattern(uint64_t i, uint64_t seed)
{
	uint64_t z = i + seed * 0x9E3779B97F4A7C15ull + 0x9E3779B97F4A7C15ull;
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

extern "C" __global__ void nvs_slab_fill(uint64_t *p, uint64_t n_words, uint64_t first_index,
					 uint64_t seed)
{
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride)
		p[i] = nvs_pattern(first_index + i, seed);
}

extern "C" __global__ void nvs_slab_verify(const uint64_t *p, uint64_t n_words,
					   uint64_t first_index, uint64_t seed,
					   unsigned long long *mismatches)
{
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	unsigned long long bad = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride)
		bad += (p[i] != nvs_pattern(first_index + i, seed));
	if (bad)
		atomicAdd(mismatches, bad);
}
