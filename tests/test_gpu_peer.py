"""Peer-HBM backing tier on real hardware (needs >= 2 GPUs with peer access;
skipped otherwise): slabs evicted from GPU 0 land in GPU 1's HBM through a
cuMemMap'ed peer allocation (no NCCL), come back bit-exact, and the traffic goes
over NVLink rather than PCIe."""
from __future__ import annotations

import pytest

pytestmark = pytest.mark.gpu

GiB = 1 << 30
MiB = 1 << 20


@pytest.fixture(scope="module")
def torch2():
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda:0")
    return torch


@pytest.mark.parametrize("fetch_v", ["tma", "ce"])
def test_evict_to_peer_hbm_and_back(torch2, artefacts, fetch_v):
    """Eviction always on the sm_90a TMA kernel; the fetch on the kernel (a fetch that has the GPU to itself)
    and on the copy engines (the default: it overlaps the previous holder's eviction kernel)."""
    torch = torch2
    from nvshare_b200 import engine as E
    size = 6 * GiB
    free1_before, _ = torch.cuda.mem_get_info(1)
    with E.Engine(peers=[1], peer_capacity_bytes=16 * GiB, peer_fetch_variant=fetch_v, elide_constant=0) as e:
        p = e.alloc(size)
        e.fetch_all()
        e.pattern_fill(p, size // 8, seed=21)
        ev = e.evict(0)
        assert ev["peer_bytes"] == size and ev["host_bytes"] == 0
        free1_out, _ = torch.cuda.mem_get_info(1)
        assert free1_before - free1_out >= size                  # the slabs live in GPU 1's HBM now
        fe = e.fetch_all()
        assert fe["peer_bytes"] == size
        assert e.pattern_verify(p, size // 8, seed=21) == 0
        evict_gbps = ev["bytes"] / 1e6 / ev["copy_ms"]
        fetch_gbps = fe["bytes"] / 1e6 / fe["copy_ms"]
        print(f"peer tier: evict (tma) {evict_gbps:.0f} GB/s, fetch ({fetch_v}) {fetch_gbps:.0f} GB/s, "
              f"kernel launches {ev['launches']}+{fe['launches']}, copy-engine calls {ev['ce_calls']}+{fe['ce_calls']}")
        assert ev["launches"] >= 1 and ev["ce_calls"] == 0
        assert (fe["launches"] >= 1 and fe["ce_calls"] == 0) if fetch_v == "tma" else fe["ce_calls"] >= 1
        assert evict_gbps > 150 and fetch_gbps > 150             # far above PCIe Gen5 x16 (~55 GB/s): NVLink
        e.free(p)


def test_peer_tier_spills_to_host(torch2, artefacts):
    from nvshare_b200 import engine as E
    with E.Engine(peers=[1], peer_capacity_bytes=2 * GiB, elide_constant=0) as e:
        p = e.alloc(3 * GiB)
        e.fetch_all()
        e.pattern_fill(p, 3 * GiB // 8, seed=4)
        ev = e.evict(0)
        assert ev["peer_bytes"] == 2 * GiB and ev["host_bytes"] == 1 * GiB
        e.fetch_all()
        assert e.pattern_verify(p, 3 * GiB // 8, seed=4) == 0
        e.free(p)
