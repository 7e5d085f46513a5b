"""The decide phase of gp_decide_tables where its warps emit ExecutorNodes and claim chunks: the index-shift emission writes
several 32-entry chunks per round (owner lanes, P loads, then the coalesced stores), and every warp starts at a fixed
chunk with only the chunks past the grid's warps claimed.  Results against the oracle (on every application of small
batches, on a sample of large ones) and against the same call with GANGPACK_TABLES=0 (every decision by the node-order
scan), for warps that mix applications with no executors, index-shift emissions and table walks, largest emitted
indices k - 1 + delta around the placement prefix length (256), uint16 and int32 outputs, batches whose chunk count is
below, near and above the number of warps the grid holds, and 2 and 16 instance groups."""
import os

import numpy as np
import pytest

from helpers import assert_same_results, group_slices, res_aos

pytestmark = pytest.mark.gpu
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
PLACE_LEN = 256                     # kPlaceLen
GRID_WARPS_H100 = 132 * 3 * 8       # an H100 SXM's decide grid: 132 SMs x 3 CTAs x 8 warps


def make_packer(gangpack, **env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return gangpack.GangPacker()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def packers(gangpack):
    ps = (make_packer(gangpack), make_packer(gangpack, GANGPACK_TABLES=0))
    yield ps
    for p in ps:
        p.close()


def roomy_cluster(rng, n_groups, per_group):
    """Nodes with room for dozens of small executors each (so counts past 256 fit), some full ones in between (zero-capacity
    runs for the walks), one executor order and one driver order per group."""
    n = n_groups * per_group
    cpu = rng.integers(2, 33, n) * 500
    mem = rng.integers(2, 65, n) * (1 << 29)
    full = rng.random(n) < 0.15
    cpu = np.where(full, rng.integers(0, 2, n) * 100, cpu).astype(np.int64)
    gpu = np.zeros(n, np.int64)
    eorder, dorder, eoff = [], [], [0]
    for g in range(n_groups):
        ids = np.arange(g * per_group, (g + 1) * per_group)
        eorder.append(rng.permutation(ids)); dorder.append(rng.permutation(ids))
        eoff.append(eoff[-1] + per_group)
    cat = lambda xs: np.concatenate(xs).astype(np.int32)
    eoff = np.array(eoff, np.int32)
    return cpu, mem, gpu, cat(eorder), cat(dorder), eoff, eoff.copy()


def mixed_apps(rng, q, n_groups):
    """Every warp mixes k = 0, small index-shift counts, counts whose k - 1 (+ the driver's displacement) is 254, 255 or
    256, and long walks; drivers with no request (delta = 0 exactly) and with one (delta > 0 where they share a node)."""
    pattern = np.array([0, 3, 255, 1, 256, 17, 257, 0, 254, 400, 2, 128, 253, 9, 600, 5], np.int32)
    count = pattern[(np.arange(q) + rng.integers(0, 16)) % 16]
    count = np.where(rng.random(q) < 0.1, rng.integers(0, 40, q), count).astype(np.int32)
    shape = rng.integers(0, 4, q)
    no_drv = rng.random(q) < 0.5
    return {
        "drv_cpu": np.where(no_drv, 0, rng.integers(1, 5, q) * 500).astype(np.int64),
        "drv_mem": np.where(no_drv, 0, rng.integers(1, 5, q) * (1 << 29)).astype(np.int64),
        "drv_gpu": np.zeros(q, np.int64),
        "exe_cpu": np.array([100, 250, 500, 125], np.int64)[shape],
        "exe_mem": np.array([1 << 27, 1 << 28, 1 << 29, 3 << 26], np.int64)[shape],
        "exe_gpu": np.zeros(q, np.int64),
        "count": count,
        "group": rng.integers(0, n_groups, q).astype(np.int32),
    }


def check_oracle(oracle, got, algo, snap, a, sel, label):
    cpu, mem, gpu, eorder, dorder, eoff, doff = snap
    dn, en, off = got
    for g in range(len(eoff) - 1):
        s = sel[a["group"][sel] == g]
        if s.size == 0:
            continue
        sub = {k: a[k][s] for k in KEYS}
        drv = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"]); exe = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
        _, wd, we, woff, _ = oracle.closed_batch(algo, 0, cpu, mem, gpu, dorder[doff[g]:doff[g + 1]], eorder[eoff[g]:eoff[g + 1]],
                                                 drv, exe, sub["count"], None)
        assert_same_results(group_slices(dn, en, off, s), (wd, we, woff), f"{label} group {g}")


def run(packers, oracle, snap, a, algo, node_bits, sample, label):
    results = []
    for p in packers:
        p.set_snapshot(*snap)
        dn, en, off = p.pack_batch(a, algo, 0, wire=dict(quantity_bits=64, node_bits=node_bits))
        results.append((dn.copy(), np.asarray(en).astype(np.int32), off))
    assert_same_results(results[0], results[1], f"{label}: tables vs scan")
    q = len(a["count"])
    rng = np.random.default_rng(q)
    sel = np.arange(q) if q <= sample else np.sort(rng.choice(q, sample, replace=False))
    check_oracle(oracle, results[0], algo, snap, a, sel, label)
    return results[0]


@pytest.mark.parametrize("n_groups", [2, 16])
@pytest.mark.parametrize("node_bits", [16, 32])
@pytest.mark.parametrize("algo", [0, 1])
def test_mixed_warps(oracle, packers, algo, node_bits, n_groups):
    rng = np.random.default_rng(1000 * algo + 10 * n_groups + node_bits)
    snap = roomy_cluster(rng, n_groups, 3000 // n_groups * 2)
    a = mixed_apps(rng, 4096, n_groups)
    dn, en, off = run(packers, oracle, snap, a, algo, node_bits, 4096, f"mixed algo {algo} bits {node_bits} groups {n_groups}")
    k = a["count"]
    placed = dn >= 0
    # the batch does exercise every emission: none, index shift (k - 1 < 256) and walks past the prefix
    assert (placed & (k == 0)).any() and (placed & (k > 0) & (k < PLACE_LEN - 1)).any()
    for kk in (255, 256, 257):
        assert (placed & (k == kk)).any(), kk
    assert (placed & (k > PLACE_LEN + 1)).any()


@pytest.mark.parametrize("q", [32, GRID_WARPS_H100 * 32 + 40, 100000])
def test_chunk_counts_around_the_grid(oracle, packers, q):
    """q = 32: one chunk, all but one warp idle; q just past the grid's warps x 32: a few claimed chunks; 100 000: the
    headline batch size, where every chunk is a warp's fixed first one on an H100."""
    rng = np.random.default_rng(q)
    snap = roomy_cluster(rng, 2, 4000)
    a = mixed_apps(rng, q, 2)
    a["count"] = np.where(rng.random(q) < 0.9, rng.integers(0, 33, q), a["count"]).astype(np.int32)
    for algo, bits in ((0, 16), (1, 32)):
        run(packers, oracle, snap, a, algo, bits, 3000, f"q={q} algo {algo} bits {bits}")
