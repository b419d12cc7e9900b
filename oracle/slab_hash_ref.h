/*
 * slab_hash_ref.h -- TEST INFRASTRUCTURE ONLY.  Plain-C restatement of the 128-bit
 * content hash the sm_90a scan kernel computes per slab (nvshare_b200/csrc/
 * slab_copy.cu, nvs_slab_scan with want_hash).  Included by the oracle
 * (oracle_slab_hash: the checker of the kernel on the GPU) and by the fake driver
 * (so that the engine's clean-slab logic runs on CPU).  No reference counterpart:
 * UVM has real dirty bits; VMM memory has none (SURVEY 8f rank 3).
 *
 * Definition: the slab is a sequence of 16-byte vectors (x, y, z, w) of 32-bit
 * little-endian words; logical lane t (0..255) owns vectors t, t+256, ... in order;
 *   a_k <- rotl32(a_k + word_k * P2, 13) * P1,   a_k(0) = SEED_k ^ (t * P1);
 * lane -> 128 bits by a bijection; slab hash = pair of 64-bit sums over the lanes.
 */
#ifndef SLAB_HASH_REF_H
#define SLAB_HASH_REF_H
#include <stdint.h>

static inline uint32_t shr_rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

static inline uint64_t shr_mix64(uint64_t z)
{
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}

static inline void slab_hash_ref(const void *slab, uint64_t bytes, uint64_t out[2])
{
	const uint32_t P1 = 0x9E3779B1u, P2 = 0x85EBCA77u;
	const uint32_t *w = (const uint32_t *)slab;
	const uint64_t n16 = bytes >> 4;
	uint64_t s0 = 0, s1 = 0;
	for (uint32_t t = 0; t < 256; ++t) {
		uint32_t a[4] = {0x243F6A88u ^ (t * P1), 0x85A308D3u ^ (t * P1), 0x13198A2Eu ^ (t * P1),
				 0x03707344u ^ (t * P1)};
		for (uint64_t i = t; i < n16; i += 256)
			for (int k = 0; k < 4; ++k)
				a[k] = shr_rotl32(a[k] + w[4 * i + k] * P2, 13) * P1;
		uint64_t u = ((uint64_t)a[0] << 32) | a[1], v = ((uint64_t)a[2] << 32) | a[3];
		u ^= (uint64_t)(t + 1) * 0x9E3779B97F4A7C15ull;
		v ^= shr_mix64(u);
		u ^= shr_mix64(v + 0xD1B54A32D192ED03ull);
		s0 += shr_mix64(u);
		s1 += shr_mix64(v);
	}
	out[0] = s0;
	out[1] = s1;
}
#endif
