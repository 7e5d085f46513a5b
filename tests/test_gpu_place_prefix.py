"""The two emission paths of gp_decide_tables at their boundary: the warp-coalesced index shift into the per-shape
placement prefix (k - 1 + delta < kPlaceLen) and the per-thread table walk (everything else), against the closed form
and the literal restatement.  The driver's node sits before, inside and after the shifted range, on a driver-only node,
in several instance groups; both packers, both output widths.  gp_last_stats.nodes_scanned (the table words read) must
equal what tests/test_place_prefix_model.py says each path reads, application by application, so both paths ran."""
import numpy as np
import pytest

from helpers import assert_same_results, group_slices, literal_batch, res_aos
from test_place_prefix_model import PLACE_LEN, emission_probes, takes_shift_path

pytestmark = pytest.mark.gpu
GI = 1 << 30
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
# per group: the prefix value S(T) (tightly-pack) / M(T) (distribute-evenly) at the first driver candidate T -- the driver's
# run lies before the boundary counts, straddles them twice, or lies after them
TARGETS = {0: (8, 250, 254, 420), 1: (8, 250, 254, 280)}
DRIVER_ONLY = 5                     # driver request (in executors) that fits only the driver-only node


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def make_case(algo, per_group=500):
    """Every group: `per_group` executor nodes of capacity 0..4 executors of (1000 m, 1 GiB) plus half a unit of slack,
    the driver order [T, X, the rest] with T an executor node of capacity 4 and X a large driver-only node."""
    rng = np.random.default_rng(11 + algo)
    caps, eorder, dorder, eoff, doff, t_pos = [], [], [], [0], [0], []
    n = 0
    for target in TARGETS[algo]:
        c = rng.integers(0, 5, per_group) * (rng.random(per_group) < 0.85)
        before = np.cumsum(c if algo == 0 else c > 0) - (c if algo == 0 else c > 0)
        assert before[-1] >= target, "the group holds fewer executors than the driver position it is built for"
        t = int(np.argmax(before >= target))
        c[t] = 4
        t_pos.append(t)
        ids = np.arange(n, n + per_group + 1)              # the last one is X
        caps.append(np.concatenate([c, [0]]))
        eorder.append(ids[:-1])
        rest = np.delete(ids[:-1], t)
        dorder.append(np.concatenate([[ids[t], ids[-1]], rest]))
        n += per_group + 1
        eoff.append(eoff[-1] + per_group); doff.append(doff[-1] + per_group + 1)
    caps = np.concatenate(caps)
    cpu = caps * 1000 + 500
    mem = caps * GI + GI // 2
    xs = np.cumsum([per_group + 1] * len(t_pos)) - 1
    cpu[xs] = 64000; mem[xs] = 64 * GI                     # X: any driver fits, it hosts no executor (not in the executor order)
    return (cpu.astype(np.int64), mem.astype(np.int64), np.zeros(n, np.int64), np.concatenate(eorder).astype(np.int32),
            np.concatenate(dorder).astype(np.int32), np.array(eoff, np.int32), np.array(doff, np.int32), caps, t_pos)


def make_apps(rng, n_groups):
    """Counts around the boundary for every driver size (delta = driver size on T for tightly-pack, 0/1 for evenly),
    plus small ones; one executor shape."""
    rows = []
    for g in range(n_groups):
        for dsz in range(DRIVER_ONLY + 1):
            for k in list(range(PLACE_LEN - 6, PLACE_LEN + 4)) + [0, 1, 2, int(rng.integers(3, 40))]:
                rows.append((g, dsz, k))
    rows = [rows[i] for i in rng.permutation(len(rows))]
    g = np.array([r[0] for r in rows], np.int32)
    dsz = np.array([r[1] for r in rows], np.int64)
    q = len(rows)
    return {"drv_cpu": dsz * 1000, "drv_mem": dsz * GI, "drv_gpu": np.zeros(q, np.int64),
            "exe_cpu": np.full(q, 1000, np.int64), "exe_mem": np.full(q, GI, np.int64), "exe_gpu": np.zeros(q, np.int64),
            "count": np.array([r[2] for r in rows], np.int32), "group": g}


def expected_table_words(algo, caps_g, t_pos, dsz, k):
    """Table words one decision reads: 2 for the driver candidate T (an executor node), then its emission."""
    c = caps_g if algo == 0 else (caps_g > 0).astype(np.int64)
    if k == 0:
        return 0
    if dsz == DRIVER_ONLY:                                  # T does not fit the driver; X is not an executor candidate
        return emission_probes(c, k, 0x7fffffff, 0, 0)
    c0 = int(c[t_pos])
    cd = int(caps_g[t_pos]) - dsz if algo == 0 else int(caps_g[t_pos] - dsz >= 1)
    return 2 + emission_probes(c, k, t_pos, c0, cd)


@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("node_bits", [32, 16])
def test_shift_and_walk_at_the_boundary(oracle, packer, algo, node_bits):
    cpu, mem, gpu, eorder, dorder, eoff, doff, caps, t_pos = make_case(algo)
    rng = np.random.default_rng(3 + algo)
    a = make_apps(rng, len(t_pos))
    packer.set_snapshot(cpu, mem, gpu, eorder, dorder, eoff, doff)
    wire = dict(quantity_bits=64, node_bits=16, offsets=False) if node_bits == 16 else None
    dn, en, off = packer.pack_batch(a, algo, 0, wire=wire) if wire else packer.pack_batch(a, algo, 0)
    en = np.asarray(en).astype(np.int32)
    st = packer.stats()
    assert st["scan_path_apps"] == 0, st

    words = 0
    paths = {True: 0, False: 0}
    for g in range(len(t_pos)):
        sel = np.nonzero(a["group"] == g)[0]
        sub = {k: a[k][sel] for k in KEYS}
        ex, dr = eorder[eoff[g]:eoff[g + 1]], dorder[doff[g]:doff[g + 1]]
        got = group_slices(dn, en, off if off is not None else np.concatenate([[0], np.cumsum(a["count"])]), sel)
        drv = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"]); exe = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
        _, wd, we, woff, _ = oracle.closed_batch(algo, 0, cpu, mem, gpu, dr, ex, drv, exe, sub["count"], None)
        assert (wd >= 0).all()                              # every decision is placed: every one emits
        assert_same_results(got, (wd, we, woff), f"closed algo {algo} group {g}")
        assert_same_results(got, literal_batch(oracle, algo, cpu, mem, gpu, dr, ex, sub), f"literal algo {algo} group {g}")
        caps_g = caps[ex]
        for dsz, k in zip(sub["drv_cpu"] // 1000, sub["count"]):
            words += expected_table_words(algo, caps_g, t_pos[g], int(dsz), int(k))
            if k and dsz != DRIVER_ONLY:
                c0 = int(caps_g[t_pos[g]]) if algo == 0 else 1
                cd = c0 - int(dsz) if algo == 0 else int(caps_g[t_pos[g]] - dsz >= 1)
                paths[takes_shift_path(int(k), c0, cd)] += 1
    assert paths[True] > 50 and paths[False] > 50, paths
    assert st["nodes_scanned"] - st["scan_path_nodes"] == words, (st, words)
