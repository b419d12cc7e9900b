/*
 * nvs_copy_desc.h -- the one data structure shared by the host engine (C) and
 * the sm_90a slab-copy kernels (CUDA).
 *
 * A descriptor is one contiguous byte move of at most one slab (2 MiB) between
 * two device-addressable ranges: local HBM (a cuMemMap'd chunk of a hooked
 * allocation), pinned host DRAM (cuMemHostAlloc DEVICEMAP, UVA) or a peer
 * GPU's HBM mapped into this context (cuMemMap of peer physical pages).
 *
 * It replaces, for this build, the implicit page list the NVIDIA UVM driver
 * builds on a GPU page fault behind the reference's single call
 * real_cuMemAllocManaged() (reference src/hook.c:673): the reference never
 * names the pages it moves; we name every slab.
 *
 * Constraints (checked by the host side, assumed by the kernels):
 *   - src, dst are 16-byte aligned
 *   - bytes is a multiple of 16 and 0 < bytes <= NVS_SLAB_BYTES
 *   - src and dst ranges of distinct descriptors in one launch do not overlap
 */
#ifndef NVS_COPY_DESC_H
#define NVS_COPY_DESC_H

#include <stdint.h>

#define NVS_SLAB_SHIFT 21u
#define NVS_SLAB_BYTES (1ull << NVS_SLAB_SHIFT) /* 2 MiB: the VMM granule and TLB page */

typedef struct nvs_copy_desc {
	uint64_t src;   /* device-addressable source address      */
	uint64_t dst;   /* device-addressable destination address */
	uint64_t bytes; /* payload bytes of this move              */
	uint64_t tag;   /* opaque to the kernel (slab id for host-side tracing) */
} nvs_copy_desc;

/* Kernel variants (see nvshare_b200/csrc/slab_copy.cu). */
enum nvs_copy_variant {
	NVS_COPY_TMA = 0, /* cp.async.bulk global->smem->global, mbarrier ring, 1 lane/warp */
	NVS_COPY_LDG = 1, /* 16-byte LDG/STG, 8-deep unroll, all lanes                  */
	NVS_COPY_CE  = 2, /* control: cuMemcpyAsync on the copy engines (no kernel)     */
};

#endif /* NVS_COPY_DESC_H */
