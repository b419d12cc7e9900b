"""Short, deterministic exercise of the copy kernels for profiling under ncu:
  1. eviction of 4 GiB to pinned host memory  (nvs_slab_copy_tma, 8 CTAs, PCIe-bound)
  2. fetch of the same with the TMA variant    (host -> HBM)
  3. a device-to-device pass over 4 GiB        (nvs_slab_copy_tma, one CTA per SM, HBM-bound)
  4. scan + splat of same-filled data          (nvs_slab_scan / nvs_slab_splat)
Numbers printed here are taken under a profiler and are NOT bench values."""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from nvshare_b200 import engine as E  # noqa: E402

GiB, MiB = 1 << 30, 1 << 20
torch.zeros(1, device="cuda")
with E.Engine(fetch_variant="tma", shared_pool_path=None) as e:
    size = 4 * GiB
    p = e.alloc(size)
    e.fetch_all()
    e.pattern_fill(p, size // 8, seed=1)
    print("evict", e.evict(0))
    print("fetch", e.fetch_all())
    q = e.alloc(size)
    e.fetch_all()
    ms = e.copy_slabs([(p + o, q + o, 2 * MiB) for o in range(0, size, 2 * MiB)], variant="tma", grid=torch.cuda.get_device_properties(0).multi_processor_count)
    print("d2d ms", ms, "GB/s payload", size / 1e6 / ms)
    t = torch.empty(1, device="cuda")
    e.free(q)
    # same-filled: fill with a constant through the splat path by evict/fetch of constant data
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
