"""Independent tightly-pack / distribute-evenly decided in one persistent launch (gp_decide_tables: classify tiles, table
segments with look-back, decide tiles, all ticket-ordered): results against the oracle and against the same call with
GANGPACK_TABLES=0 (every decision by the node-order scan), at the shapes where the work items meet -- group sizes at the
segment boundaries, empty groups, hundreds of groups, batches around the 32-application threshold, more shapes than
tables, offsets derived on the device over many tiles, three pipeline lanes at once, graph replay, and the zone entry
points that run the same launch."""
import os

import numpy as np
import pytest

from helpers import assert_same_results, group_slices, random_apps, random_cluster, res_aos

pytestmark = pytest.mark.gpu
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
SEG = 1024                          # nodes per table segment (kTabSeg)


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


def grouped_cluster(rng, sizes, tight=False):
    """One instance group per entry of `sizes` (executor-order length); the driver order of a group is a permutation of its
    executor candidates plus two driver-only nodes."""
    n_exec = int(sum(sizes))
    n = n_exec + 2 * len(sizes)
    cpu, mem, gpu = random_cluster(rng, n, tight=tight)
    eorder, dorder, eoff, doff = [], [], [0], [0]
    base = 0
    for k, sz in enumerate(sizes):
        ex = np.arange(base, base + sz)
        base += sz
        drv_only = np.array([n_exec + 2 * k, n_exec + 2 * k + 1])
        eorder.append(rng.permutation(ex))
        dorder.append(rng.permutation(np.concatenate([ex, drv_only])))
        eoff.append(eoff[-1] + sz); doff.append(doff[-1] + sz + 2)
    cat = lambda xs: np.concatenate(xs).astype(np.int32)
    return cpu, mem, gpu, cat(eorder), cat(dorder), np.array(eoff, np.int32), np.array(doff, np.int32)


def few_shape_apps(rng, q, n_groups, n_shapes=6):
    a = random_apps(rng, q, big_counts=True)
    s = rng.integers(0, n_shapes, q)
    a["exe_cpu"] = np.array([250, 500, 750, 1000, 1500, 2000, 300, 900], np.int64)[s % 8]
    a["exe_mem"] = np.array([1 << 28, 3 << 28, 1 << 29, 1 << 30, (1 << 30) + 7, 1 << 31, 5 << 27, 7 << 27], np.int64)[s % 8]
    a["group"] = rng.integers(0, n_groups, q).astype(np.int32)
    return a


def check_against_oracle(oracle, got, algo, cpu, mem, gpu, eorder, dorder, eoff, doff, a, label, groups=None):
    dn, en, off = got
    for g in (range(len(eoff) - 1) if groups is None else groups):
        sel = np.nonzero(a["group"] == g)[0]
        if sel.size == 0:
            continue
        sub = {k: a[k][sel] for k in KEYS}
        ex, dr = eorder[eoff[g]:eoff[g + 1]], dorder[doff[g]:doff[g + 1]]
        drv = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"]); exe = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
        _, wd, we, woff, _ = oracle.closed_batch(algo, 0, cpu, mem, gpu, dr, ex, drv, exe, sub["count"], None)
        assert_same_results(group_slices(dn, en, off, sel), (wd, we, woff), f"{label} group {g}")


def run_both(packers, snap, a, algo, **kw):
    got = []
    for p in packers:
        p.set_snapshot(*snap)
        dn, en, off = p.pack_batch(a, algo, 0, **kw)
        got.append((dn.copy(), np.asarray(en).astype(np.int32), off, p.stats()))
    assert_same_results(got[0][:3], got[1][:3], f"tables vs scan algo {algo}")
    return got[0]


@pytest.mark.parametrize("algo", [0, 1])
def test_group_sizes_at_segment_boundaries(oracle, packers, algo):
    rng = np.random.default_rng(100 + algo)
    sizes = [0, 1, SEG - 1, SEG, SEG + 1, 2 * SEG, 3 * SEG + 5, 0, 7]
    snap = grouped_cluster(rng, sizes)
    a = few_shape_apps(rng, 4000, len(sizes))
    dn, en, off, st = run_both(packers, snap, a, algo)
    assert st["scan_path_apps"] < len(dn) // 2, st
    check_against_oracle(oracle, (dn, en, off), algo, *snap, a, f"segments algo {algo}")


@pytest.mark.parametrize("algo", [0, 1])
def test_hundreds_of_groups(oracle, packers, algo):
    rng = np.random.default_rng(300 + algo)
    sizes = list(rng.integers(0, 12, 330))
    snap = grouped_cluster(rng, sizes, tight=True)
    a = few_shape_apps(rng, 3000, len(sizes))
    dn, en, off, _ = run_both(packers, snap, a, algo)
    check_against_oracle(oracle, (dn, en, off), algo, *snap, a, f"330 groups algo {algo}", groups=range(0, 330, 11))


@pytest.mark.parametrize("q", [1, 31, 32, 33])
def test_batch_sizes_around_the_table_threshold(oracle, packers, q):
    rng = np.random.default_rng(q)
    snap = grouped_cluster(rng, [600, 1500])
    a = few_shape_apps(rng, q, 2)
    for algo in (0, 1):
        dn, en, off, _ = run_both(packers, snap, a, algo)
        check_against_oracle(oracle, (dn, en, off), algo, *snap, a, f"q={q} algo {algo}")


def test_more_shapes_than_tables(oracle, packers):
    rng = np.random.default_rng(65)
    snap = grouped_cluster(rng, [2500, 900])
    a = few_shape_apps(rng, 3000, 2)
    a["exe_mem"] = a["exe_mem"] + rng.integers(0, 200, 3000) * (1 << 20)
    for algo in (0, 1):
        dn, en, off, st = run_both(packers, snap, a, algo)
        assert 0 < st["scan_path_apps"] < 3000, st
        check_against_oracle(oracle, (dn, en, off), algo, *snap, a, f"many shapes algo {algo}")


def test_offsets_derived_over_many_tiles(gangpack, packers):
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(5000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    apps = synth.make_apps(150000)
    a = {k: apps[k] for k in KEYS}
    a["count"] = np.where(np.arange(150000) % 97 == 0, 0, a["count"]).astype(np.int32)
    snap = (nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    for algo in (0, 1):
        ref = run_both(packers, snap, a, algo)[:3]
        for p in packers:
            got = p.pack_batch(a, algo, 0, wire=dict(quantity_bits=64, node_bits=32, offsets=False))
            assert_same_results((got[0], np.asarray(got[1]).astype(np.int32), got[2]), ref, f"derived offsets algo {algo}")


def test_three_pipeline_lanes_and_graph_replay(gangpack, packers):
    """Small chunks: consecutive chunks run their launches concurrently on the three lanes; the same call repeated until
    the chunk graphs are replayed gives the same bits every time."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(4000, groups=3)
    eoff, eorder = synth.group_orders(nodes)
    apps = synth.make_apps(24000, groups=3)
    a = {k: apps[k] for k in KEYS + ("group",)}
    snap = (nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    p = make_packer(gangpack, GANGPACK_CHUNK_APPS=2048)
    try:
        for algo in (0, 1):
            ref = run_both(packers, snap, a, algo)[:3]
            p.set_snapshot(*snap)
            pin = p.pinned_columns(len(a["count"]), [k for k in KEYS if k != "count"] + ["group"], dtype=np.int64)
            for k in pin:
                pin[k][:] = a[k]
            pin["group"] = p.pinned(len(a["count"]), np.int32); pin["group"][:] = a["group"]
            pin["count"] = p.pinned(len(a["count"]), np.int32); pin["count"][:] = a["count"]
            for rep in range(5):
                got = p.pack_batch(pin, algo, 0)
                assert_same_results((got[0], np.asarray(got[1]).astype(np.int32), got[2]), ref, f"chunked algo {algo} call {rep}")
                got = p.pack_batch(a, algo, 0)
                assert_same_results((got[0], np.asarray(got[1]).astype(np.int32), got[2]), ref, f"pageable algo {algo} call {rep}")
    finally:
        p.close()


def test_zone_entry_points(packers):
    """gp_pack_batch_zones and gp_pack_batch_az_aware (whose undivided fallback is the independent batch) give the same
    bits with the tables and with the scan."""
    rng = np.random.default_rng(70)
    Z, per = 70, 3
    n = (Z + 1) * per
    cpu, mem, gpu = random_cluster(rng, n)
    sc, sm = cpu + rng.integers(0, 9, n) * 250, mem + rng.integers(0, 17, n) * (1 << 28)
    zone_of = rng.permutation(np.arange(n) % (Z + 1))
    order_all = rng.permutation(n).astype(np.int32)
    eo, eoff = [], [0]
    for z in range(Z + 1):                                  # zone Z: the trailing group of the az-aware layout
        eo += [int(i) for i in order_all if zone_of[i] == z]
        eoff.append(len(eo))
    eo = np.array(eo, np.int32); eoff = np.array(eoff, np.int32)
    apps = random_apps(rng, 400)
    apps["count"] = np.where(rng.random(400) < 0.2, rng.integers(10, 40, 400), apps["count"]).astype(np.int32)
    outs = []
    for p in packers:
        p.set_snapshot(cpu, mem, gpu, eo[:eoff[Z]], eo[:eoff[Z]], eoff[:Z + 1], eoff[:Z + 1])
        p.set_schedulable(sc, sm, gpu.clip(0))
        z1 = [x.copy() for x in p.pack_batch_zones(apps, 0)]
        p.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
        p.set_schedulable(sc, sm, gpu.clip(0))
        z2 = [x.copy() for x in p.pack_batch_az_aware(apps, order_all, order_all, Z)]
        outs.append((z1, z2))
    (a1, a2), (b1, b2) = outs
    for x, y in zip(a1 + a2, b1 + b2):
        assert np.array_equal(x, y)
