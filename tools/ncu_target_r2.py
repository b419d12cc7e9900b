"""Round 2: short, deterministic exercise of the sm_90a kernels for profiling under ncu:
  1. eviction of 4 GiB of position-dependent data: nvs_slab_scan (hash mode, one launch over 2048 slabs,
     HBM-bound) + copy engines; fetch; a second eviction that finds everything clean (scan only)
  2. a device-to-device pass over 4 GiB (nvs_slab_copy_tma, one CTA per SM, HBM-bound)
  3. with --peer: eviction / fetch of 4 GiB to the HBM of GPU 1 (nvs_slab_copy_tma over NVLink, half the SMs)
  4. scan + splat of same-filled data (nvs_slab_scan quick mode / nvs_slab_splat)
Numbers printed here are taken under a profiler and are NOT bench values."""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from nvshare_b200 import engine as E  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
peer = "--peer" in sys.argv
torch.zeros(1, device="cuda")
kw = dict(shared_pool_path=None, batch_bytes=4 * GiB)
if peer:
    kw.update(peers=[1], peer_capacity_bytes=16 * GiB, peer_fetch_variant="tma")
with E.Engine(**kw) as e:
    size = 4 * GiB
    p = e.alloc(size)
    e.fetch_all()
    e.pattern_fill(p, size // 8, seed=1)
    print("evict", e.evict(0))
    print("fetch", e.fetch_all())
    print("evict(clean)", e.evict(0))
    print("fetch", e.fetch_all())
    q = e.alloc(size)
    e.fetch_all()
    ms = e.copy_slabs([(p + o, q + o, 2 * MiB) for o in range(0, size, 2 * MiB)], variant="tma", grid=torch.cuda.get_device_properties(0).multi_processor_count)
    print("d2d ms", ms, "GB/s payload", size / 1e6 / ms)
    e.free(q)

    class Raw:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}
    x = torch.as_tensor(Raw(p, size // 4), device="cuda")
    x.fill_(1.0)
    torch.cuda.synchronize()
    print("evict(ones)", e.evict(0))
    print("fetch(ones)", e.fetch_all())
    del x
    e.free(p)
