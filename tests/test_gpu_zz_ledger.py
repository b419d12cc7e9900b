"""The GPU ledger (nvshare_b200/csrc/gpu_ledger.c) on the real driver.  Its rules are pinned on the fake
driver's four GPUs (test_gpu_ledger_fake.py); here: that the ledger comes up on an H100 at all (the UUID and
the total come from the driver), that the engine's own footprint is on record where other processes can see
it and leaves with the memory, and -- on a box with two GPUs -- that what an engine backs on GPU 1 is
accounted on GPU 1 while it is there."""
from __future__ import annotations

import pytest

pytestmark = pytest.mark.gpu

GiB = 1 << 30
MiB = 1 << 20


@pytest.fixture(scope="module")
def torch0():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda:0")
    return torch


def test_own_footprint_is_on_record_and_leaves_with_the_memory(torch0, artefacts):
    from nvshare_b200 import engine as E
    _, total = torch0.cuda.mem_get_info(0)
    with E.Engine() as e:
        acc = e.gpu_account(-1)
        assert acc["tracked"] == 1 and acc["device"] == 0
        assert acc["total_bytes"] == total                       # cuDeviceTotalMem == cuMemGetInfo's total
        assert acc["reserve_bytes"] == 1536 * MiB                # the slice the reference hides too (src/hook.c:45)
        before = acc["my_own_bytes"]
        p = e.alloc(512 * MiB)
        acc = e.gpu_account(-1)
        assert acc["my_own_bytes"] == before + 512 * MiB and acc["max_own_bytes"] >= acc["my_own_bytes"]
        assert acc["lent_bytes"] == 0 and e.gpu_lent_bytes() == 0    # nobody backs anything on this GPU
        e.fetch_all()
        e.pattern_fill(p, 512 * MiB // 8, seed=5)
        e.evict(0)                                               # swapped out or not: the claim is the footprint
        assert e.gpu_account(-1)["my_own_bytes"] == before + 512 * MiB
        e.fetch_all()
        assert e.pattern_verify(p, 512 * MiB // 8, seed=5) == 0
        e.free(p)
        assert e.gpu_account(-1)["my_own_bytes"] == before


def test_backing_on_a_peer_is_accounted_on_that_peer(torch0, artefacts):
    if torch0.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from nvshare_b200 import engine as E
    size = 4 * GiB
    with E.Engine(peers=[1], peer_capacity_bytes=16 * GiB, elide_constant=0) as e:
        peer = e.gpu_account(0)
        assert peer["tracked"] == 1 and peer["device"] == 1 and peer["my_lent_bytes"] == 0
        p = e.alloc(size)
        e.fetch_all()
        e.pattern_fill(p, size // 8, seed=9)
        ev = e.evict(0)
        assert ev["peer_bytes"] == size
        peer = e.gpu_account(0)
        assert size <= peer["my_lent_bytes"] <= peer["lent_bytes"] and peer["refusals"] == 0    # whole arenas
        assert e.gpu_account(-1)["lent_bytes"] == 0              # GPU 0 itself lends nothing
        e.fetch_all()
        assert e.pattern_verify(p, size // 8, seed=9) == 0
        assert e.gpu_account(0)["my_lent_bytes"] == 0            # empty arenas go back at once
        e.free(p)


def test_peers_auto_on_whatever_this_box_has(torch0, artefacts):
    """NVSHARE_PEERS=auto: with one GPU there is no peer and everything goes to pinned host memory; with more,
    the other GPUs hold it (they are idle here, the ledger lets them lend)."""
    from nvshare_b200 import engine as E
    size = 1 * GiB
    with E.Engine(peers="auto", elide_constant=0) as e:
        p = e.alloc(size)
        e.fetch_all()
        e.pattern_fill(p, size // 8, seed=13)
        ev = e.evict(0)
        assert ev["bytes"] + ev["clean_bytes"] == size
        if torch0.cuda.device_count() > 1:
            assert ev["peer_bytes"] == size and e.gpu_account(0)["tracked"] == 1
        else:
            assert ev["peer_bytes"] == 0
        e.fetch_all()
        assert e.pattern_verify(p, size // 8, seed=13) == 0
        e.free(p)
