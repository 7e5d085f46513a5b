"""gp_destroy returns every device buffer of its context.  Each cycle creates a context, lays out a 2 000-group snapshot,
packs one independent tightly-pack batch large enough to take the capacity-table path (which reserves the per-shape
placement prefixes, about 64 KB per instance group and lane) and destroys the context.  After a warm-up cycle, four more
cycles must leave the device's free memory where it was."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
N_GROUPS = 2000
NODES_PER_GROUP = 3
N_APPS = 64                 # >= 32: the table path
CYCLES = 4
SLACK = 64 << 20            # bytes; a leaked placement prefix alone is ~160 MB per cycle at 2 000 groups
GI = 1 << 30


@pytest.fixture(scope="module")
def gangpack_lib():
    import k8s_spark_scheduler_b200 as g
    g.native.load()
    return g


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    torch.cuda.init()
    return torch


def make_case():
    n = N_GROUPS * NODES_PER_GROUP
    order = np.arange(n, dtype=np.int32)
    off = np.arange(0, n + 1, NODES_PER_GROUP, dtype=np.int32)
    nodes = (np.full(n, 8000, np.int64), np.full(n, 32 * GI, np.int64), np.zeros(n, np.int64), order, order, off, off)
    apps = {"drv_cpu": np.full(N_APPS, 1000, np.int64), "drv_mem": np.full(N_APPS, GI, np.int64),
            "drv_gpu": np.zeros(N_APPS, np.int64), "exe_cpu": np.full(N_APPS, 1000, np.int64),
            "exe_mem": np.full(N_APPS, GI, np.int64), "exe_gpu": np.zeros(N_APPS, np.int64),
            "count": np.full(N_APPS, 2, np.int32), "group": (np.arange(N_APPS) * 31 % N_GROUPS).astype(np.int32)}
    return nodes, apps


def cycle(g, nodes, apps):
    p = g.GangPacker(device=0)
    try:
        p.set_snapshot(*nodes)
        driver, _, _ = p.pack_batch(apps, g.TIGHTLY_PACK, g.MODE_INDEPENDENT)
        assert (driver >= 0).all(), "every application fits its group"
    finally:
        p.close()


def test_destroy_frees_device_memory(gangpack_lib, torch_cuda, monkeypatch):
    monkeypatch.delenv("GANGPACK_TABLES", raising=False)      # the table path reserves the placement prefixes
    nodes, apps = make_case()
    cycle(gangpack_lib, nodes, apps)                          # warm-up: module loads, torch's own context
    torch_cuda.cuda.synchronize()
    free_before = torch_cuda.cuda.mem_get_info(0)[0]
    for _ in range(CYCLES):
        cycle(gangpack_lib, nodes, apps)
    torch_cuda.cuda.synchronize()
    free_after = torch_cuda.cuda.mem_get_info(0)[0]
    dropped = free_before - free_after
    print(f"free device memory dropped by {dropped / 2**20:.1f} MiB over {CYCLES} context cycles")
    assert dropped < SLACK, f"{CYCLES} create/pack/destroy cycles lost {dropped / 2**20:.1f} MiB of device memory"
