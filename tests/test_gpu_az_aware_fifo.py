"""gp_pack_fifo_az_aware = fitEarlierDrivers (resource.go:224-262) with AzAwareTightlyPack (az_aware_pack_tightly.go:27-38)
as BinpackFunc, the whole queue in one launch: every zone is packed with tightly-pack and chosen by packing efficiency
like gp_pack_fifo_zones, and when no zone wins the undivided fallback (SparkBinPack + tightlyPackExecutors over the full
driver / executor orders) runs on the device against the availability the loop holds at that point.

Every case runs both accounting modes against the literal restatement's loop (orc_fifo with the az-aware packer over the
undivided orders): every driver_node (including -1 / -2), every ExecutorNodes slice and the availability left behind.
Small cases also walk the queue with the pure-Python statement to check which applications a zone won and which the
fallback decided, and gp_stats.scan_path_apps counts the latter."""
import numpy as np
import pytest

from helpers import node_names, random_apps, random_cluster, res_aos
from oracle import pyref

pytestmark = pytest.mark.gpu

ORC_AZ_AWARE = 3


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def az_layout(order_d, order_e, zone_of):
    """What a shim uploads for gp_pack_fifo_az_aware: one group per candidate zone (driverZonesInOrder order, zones without
    executor candidates left out, single_az.go:36-41) holding the undivided orders restricted to that zone, then one
    trailing group with every other node of the two orders.  -> (zones, exec_order, drv_order, exec_off, drv_off)."""
    zones, dz, ez = [], {}, {}
    for n in order_d:
        z = zone_of[n]
        if z not in dz:
            zones.append(z); dz[z] = []
        dz[z].append(n)
    for n in order_e:
        ez.setdefault(zone_of[n], []).append(n)
    zones = [z for z in zones if z in ez]
    eoff, doff, eo, do = [0], [0], [], []
    for z in zones:
        eo += ez[z]; do += dz[z]
        eoff.append(len(eo)); doff.append(len(do))
    cand = set(zones)
    te = [n for n in order_e if zone_of[n] not in cand]
    td = [n for n in order_d if zone_of[n] not in cand]
    if te or td or not zones:
        eo += te; do += td
        eoff.append(len(eo)); doff.append(len(do))
    return zones, np.array(eo, np.int32), np.array(do, np.int32), np.array(eoff, np.int32), np.array(doff, np.int32)


def run_case(oracle, packer, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, label, walk=True):
    """Both accounting modes: device vs the literal loop (and, with `walk`, the zone / fallback split vs pyref).
    -> [(mode, zone, driver_node, executor_nodes, off, stats)]."""
    n = len(cpu)
    names = node_names(n)
    labels = ["zone-%d" % z for z in zone_of]
    zones, eo, do, eoff, doff = az_layout(order_d, order_e, zone_of)
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"]); exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    dnames = [names[i] for i in order_d]; enames = [names[i] for i in order_e]
    runs = []
    for mode in (1, 2):
        cl = oracle.Cluster(names, cpu, mem, gpu, sched=(sc, sm, sg), zone=labels)
        _, wd, we, woff = cl.fifo(ORC_AZ_AWARE, mode, drv, exe, apps["count"], apps["young"], dnames, enames, with_efficiencies=True)
        packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
        packer.set_schedulable(sc, sm, sg)
        zone, gd, ge, goff, avg = packer.pack_fifo_az_aware(apps, mode, order_e, order_d, len(zones))
        st = packer.stats()
        assert np.array_equal(goff, woff)
        bad = np.nonzero(gd != wd)[0]
        assert bad.size == 0, (label, mode, bad[:5], gd[bad[:5]], wd[bad[:5]], zone[bad[:5]])
        for i in np.nonzero(wd >= 0)[0]:
            assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]]), (label, mode, i)
        fc, fm, fg = packer.get_snapshot()
        wc, wm, wg = cl.available()
        assert np.array_equal(fc, wc) and np.array_equal(fm, wm) and np.array_equal(fg, wg), (label, mode)
        # zone -1 + a driver = the fallback placed it, with zero averages; a zone winner has a positive average
        assert (zone[gd < 0] == -1).all()
        assert (avg[(zone == -1)] == 0.0).all()
        assert (avg[zone >= 0, 3] > 0.0).all()
        evaluated = gd != -2
        assert st["scan_path_apps"] == int((evaluated & (zone == -1)).sum()), (label, mode, st)
        if walk and n < 400:
            _walk(names, cpu, mem, gpu, sc, sm, sg, labels, dnames, enames, zones, apps, mode, zone, gd, ge, goff, label)
        runs.append((mode, zone, gd, ge, goff, st))
    return runs


def _walk(names, cpu, mem, gpu, sc, sm, sg, labels, dnames, enames, zones, apps, mode, zone, gd, ge, goff, label):
    """The queue in pure Python: zone[i] is the winning zone when single_az_tightly_pack succeeds on the state before
    application i, and -1 (fallback) otherwise; the fallback's placement is pyref's az_aware_tightly_pack."""
    meta = {names[i]: (int(cpu[i]), int(mem[i]), int(gpu[i])) for i in range(len(names))}
    sched = {names[i]: (int(sc[i]), int(sm[i]), int(sg[i])) for i in range(len(names))}
    zmap = dict(zip(names, labels))
    zlabels = ["zone-%d" % z for z in zones]
    for i in range(len(apps["count"])):
        if gd[i] == -2:
            break
        d_req = (int(apps["drv_cpu"][i]), int(apps["drv_mem"][i]), int(apps["drv_gpu"][i]))
        e_req = (int(apps["exe_cpu"][i]), int(apps["exe_mem"][i]), int(apps["exe_gpu"][i]))
        k = int(apps["count"][i])
        d, ex, ok = pyref.single_az_tightly_pack(d_req, e_req, k, dnames, enames, meta, sched, zmap)
        if ok:
            assert zone[i] == zlabels.index(zmap[d]), (label, mode, i)
        else:
            assert zone[i] == -1, (label, mode, i)
            d, ex, ok = pyref.az_aware_tightly_pack(d_req, e_req, k, dnames, enames, meta, sched, zmap)
        assert ok == (gd[i] >= 0), (label, mode, i)
        if not ok:
            continue
        assert names[gd[i]] == d and [names[j] for j in ge[goff[i]:goff[i + 1]]] == ex, (label, mode, i)
        if mode == 1:
            for nm, u in pyref.spark_resource_usage(d_req, e_req, d, ex).items():
                meta[nm] = pyref.sub(meta[nm], u)
        else:
            meta[d] = pyref.sub(meta[d], d_req)
            for nm in ex:
                meta[nm] = pyref.sub(meta[nm], e_req)


def _random_case(seed):
    rng = np.random.default_rng(8800 + seed)
    n = int(rng.integers(40, 200)); Z = int(rng.integers(1, 6)); q = 220
    cpu, mem, gpu = random_cluster(rng, n, tight=bool(seed % 2), gpus=bool(seed % 3 == 0))
    sc = cpu + rng.integers(0, 9, n) * 250 + (rng.integers(0, 3, n) == 0) * 1
    sm = mem + rng.integers(0, 17, n) * (1 << 28)
    sg = np.maximum(gpu, 0) + (rng.integers(0, 2, n) if seed % 3 == 0 else 0)
    p = rng.random(Z) ** 2 + 0.05                                      # zones of unequal size
    zone_of = rng.choice(Z, size=n, p=p / p.sum())
    order_e = [int(i) for i in rng.permutation(n) if rng.random() < 0.9]
    order_d = [int(i) for i in rng.permutation(n)[: max(1, int(n * 0.7))]]
    apps = random_apps(rng, q, gpus=bool(seed % 3 == 0), zero_dims=bool(seed == 5))
    big = rng.random(q) < 0.12                                          # larger than any one zone can hold
    apps["count"] = np.where(big, rng.integers(20, 90, q), apps["count"]).astype(np.int32)
    apps["young"] = (rng.random(q) < (0.97 if seed % 2 else 1.0)).astype(np.uint8)
    return cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps


@pytest.mark.parametrize("seed", range(6))
def test_az_aware_fifo_randomized(oracle, packer, seed):
    case = _random_case(seed)
    runs = run_case(oracle, packer, *case, label=f"seed {seed}")
    for mode, zone, gd, _, _, st in runs:
        assert st["scan_path_apps"] > 0, (seed, mode)                 # the fallback ran


def _apps(rows, young=None):
    """rows: (drv_cpu, drv_mem, exe_cpu, exe_mem, count)"""
    r = np.array(rows, np.int64).reshape(-1, 5)
    q = len(r)
    return {"drv_cpu": r[:, 0], "drv_mem": r[:, 1], "drv_gpu": np.zeros(q, np.int64), "exe_cpu": r[:, 2], "exe_mem": r[:, 3],
            "exe_gpu": np.zeros(q, np.int64), "count": r[:, 4].astype(np.int32),
            "young": np.ones(q, np.uint8) if young is None else np.array(young, np.uint8)}


G = 1 << 30
# zone 0: nodes 0-1 (driver + executor candidates); zone 1: node 2, driver candidate only; zone 2: nodes 3-5, executor
# candidates only; zone 3: nodes 6-7 (driver + executor candidates, the second candidate zone)
CPU8 = np.array([4000, 4000, 12000, 4000, 4000, 4000, 4000, 4000], np.int64)
MEM8 = np.full(8, 64 * G, np.int64)
ZONE8 = np.array([0, 0, 1, 2, 2, 2, 3, 3])
ORDER_E8 = [3, 0, 4, 1, 6, 5, 7]
ORDER_D8 = [2, 0, 6, 1, 7]


def _constructed(oracle, packer, apps, label, cpu=CPU8, sc=None):
    n = len(cpu)
    sc = cpu + 4000 if sc is None else sc
    return run_case(oracle, packer, cpu, MEM8[:n], np.zeros(n, np.int64), sc, MEM8[:n] + 8 * G, np.zeros(n, np.int64),
                    ZONE8[:n], ORDER_D8, ORDER_E8, apps, label)


def test_fallback_spans_zones(oracle, packer):
    """The driver only fits on the driver-only zone's node, so no zone wins; the fallback puts it there and its executors on
    the executor-only zone's nodes and zone 0's, in the undivided order.  exe_count 0 takes the same path."""
    apps = _apps([(6000, G, 2000, G, 6), (5000, G, 1000, G, 0)])
    runs = _constructed(oracle, packer, apps, "spans zones")
    for mode, zone, gd, ge, goff, st in runs:
        assert list(zone) == [-1, -1] and list(gd) == [2, 2] and st["scan_path_apps"] == 2
        assert list(ge[goff[0]:goff[1]]) == [3, 3, 0, 0, 4, 4]         # driver in zone 1, executors in zones 2 and 0


def test_fallback_changes_the_next_zone_choice(oracle, packer):
    """Zone 0 would win the second application on its own (a tie with zone 3 goes to the first zone); after the fallback
    charged zone 0's nodes, zone 0 cannot host it and zone 3 wins."""
    alone = _apps([(1000, G, 1000, G, 6)])
    zone_alone = _constructed(oracle, packer, alone, "alone")[0][1]
    both = _apps([(6000, G, 2000, G, 6), (1000, G, 1000, G, 6)])
    runs = _constructed(oracle, packer, both, "after fallback")
    for mode, zone, gd, _, _, _ in runs:
        assert zone_alone[0] == 0 and zone[0] == -1 and gd[0] >= 0 and zone[1] == 1, (mode, zone, gd)


@pytest.mark.parametrize("young", [0, 1])
def test_fallback_that_fits_nowhere(oracle, packer, young):
    apps = _apps([(1000, G, 1000, G, 1), (6000, G, 4000, G, 40), (1000, G, 1000, G, 1)], young=[1, young, 1])
    runs = _constructed(oracle, packer, apps, f"nowhere young={young}")
    for mode, zone, gd, _, _, st in runs:
        assert gd[0] >= 0 and gd[1] == -1 and zone[1] == -1
        assert (gd[2] >= 0) if young else (gd[2] == -2)
        assert st["scan_path_apps"] == 1


@pytest.mark.parametrize("count", [65535, 65536, 70000])
def test_large_counts_across_zones(oracle, packer, count):
    """One executor per milli-core: every zone holds fewer than `count`, the whole cluster holds them (the k > 0xFFFF
    scan without the capacity cache)."""
    n = 8
    cpu = np.full(n, 12000, np.int64)
    apps = _apps([(500, 1, 1, 1, count), (500, 1, 1, 1, 3)])
    runs = run_case(oracle, packer, cpu, MEM8, np.zeros(n, np.int64), cpu + 1000, MEM8 + G, np.zeros(n, np.int64),
                    ZONE8, ORDER_D8, ORDER_E8, apps, f"count {count}", walk=False)
    for mode, zone, gd, _, _, st in runs:
        assert zone[0] == -1 and gd[0] >= 0 and st["scan_path_apps"] >= 1


def test_general_class_and_negative_gpu(oracle, packer):
    """Requests and availabilities of 2^32 and more (the general arithmetic class) and negative gpu availabilities."""
    rng = np.random.default_rng(77)
    n, q = 90, 160
    cpu, mem, gpu = random_cluster(rng, n, gpus=True, negative=True)
    mem = mem * 37 + (1 << 41)
    sc, sm, sg = np.abs(cpu) + 8000, mem + (1 << 40), np.maximum(gpu, 0) + 1
    zone_of = rng.integers(0, 4, n)
    order_e = [int(i) for i in rng.permutation(n) if rng.random() < 0.85]
    order_d = [int(i) for i in rng.permutation(n)[:60]]
    apps = random_apps(rng, q, gpus=True)
    apps["exe_mem"] = apps["exe_mem"] * 41 + (1 << 33) + 7
    apps["drv_mem"] = apps["drv_mem"] * 3 + (1 << 32)
    apps["count"] = np.where(rng.random(q) < 0.15, rng.integers(15, 60, q), apps["count"]).astype(np.int32)
    apps["young"] = np.ones(q, np.uint8)
    runs = run_case(oracle, packer, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, "general class")
    assert all(st["scan_path_apps"] > 0 for *_, st in runs)


def test_64_zones_and_a_trailing_group(oracle, packer):
    rng = np.random.default_rng(64)
    Z, per = 66, 3
    n = Z * per
    cpu, mem, gpu = random_cluster(rng, n)
    sc, sm = cpu + rng.integers(0, 9, n) * 250, mem + rng.integers(0, 17, n) * (1 << 28)
    zone_of = rng.permutation(np.arange(n) % Z)
    order_e = [int(i) for i in rng.permutation(n) if zone_of[i] != 64]            # zone 64: driver candidates only
    order_d = [int(i) for i in rng.permutation(n) if zone_of[i] != 65]            # zone 65: executor candidates only
    apps = random_apps(rng, 150)
    apps["count"] = np.where(rng.random(150) < 0.2, rng.integers(10, 40, 150), apps["count"]).astype(np.int32)
    apps["young"] = (rng.random(150) < 0.97).astype(np.uint8)
    zones = az_layout(order_d, order_e, zone_of)[0]
    assert len(zones) == 64
    runs = run_case(oracle, packer, cpu, mem, gpu, sc, sm, gpu.clip(0), zone_of, order_d, order_e, apps, "64 zones")
    for mode, zone, gd, _, _, st in runs:
        assert (zone >= 16).any() and st["scan_path_apps"] > 0


@pytest.mark.parametrize("mode", [1, 2])
def test_no_candidate_zone_is_plain_fifo_tightly_pack(oracle, packer, mode):
    """n_zones = 0 (no zone has both kinds of candidates): every application takes the fallback, which is then
    gp_pack_batch in the same FIFO mode with tightly-pack on the undivided one-group snapshot."""
    rng = np.random.default_rng(500 + mode)
    n = 120
    cpu, mem, gpu = random_cluster(rng, n)
    zone_of = np.where(np.arange(n) % 2 == 0, 0, 1)
    order_e = [int(i) for i in rng.permutation(n) if zone_of[i] == 0]
    order_d = [int(i) for i in rng.permutation(n) if zone_of[i] == 1]
    apps = random_apps(rng, 200)
    apps["young"] = (rng.random(200) < 0.98).astype(np.uint8)
    runs = run_case(oracle, packer, cpu, mem, gpu, cpu + 1000, mem + G, gpu, zone_of, order_d, order_e, apps, "no zones")
    for _, zone, gd, _, _, st in runs:
        assert (zone == -1).all() and st["scan_path_apps"] == int((gd != -2).sum()) > 0
    zones, eo, do, eoff, doff = az_layout(order_d, order_e, zone_of)
    assert zones == [] and len(eoff) == 2
    packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    packer.set_schedulable(cpu + 1000, mem + G, gpu)
    _, gd, ge, goff, _ = packer.pack_fifo_az_aware(apps, mode, order_e, order_d, 0)
    after = packer.get_snapshot()
    packer.set_snapshot(cpu, mem, gpu, order_e, order_d)
    bd, be, boff = packer.pack_batch(apps, 0, mode)
    assert np.array_equal(bd, gd)
    for i in np.nonzero(gd >= 0)[0]:
        assert np.array_equal(be[boff[i]:boff[i + 1]], ge[goff[i]:goff[i + 1]])
    for x, y in zip(packer.get_snapshot(), after):
        assert np.array_equal(x, y)


def test_hand_off_to_a_zone_batch(oracle, packer):
    """After the loop the device holds the charged availability: a gp_pack_batch_zones on the same context sees it."""
    rng = np.random.default_rng(31)
    n = 80
    cpu, mem, gpu = random_cluster(rng, n)
    sc, sm = cpu + 4000, mem + 8 * G
    zone_of = np.arange(n) % 3
    order = [int(i) for i in rng.permutation(n)]
    apps = random_apps(rng, 60)
    apps["count"][::7] = 120
    apps["young"] = np.ones(60, np.uint8)
    names = node_names(n)
    runs = run_case(oracle, packer, cpu, mem, gpu, sc, sm, gpu, zone_of, order, order, apps, "hand-off")
    assert runs[-1][5]["scan_path_apps"] > 0
    fc, fm, fg = packer.get_snapshot()                                  # exact accounting ran last
    nxt = random_apps(rng, 50)
    zone, gd, ge, goff, _ = packer.pack_batch_zones(nxt, 0)
    cl = oracle.Cluster(names, fc, fm, fg, sched=(sc, sm, gpu), zone=["zone-%d" % z for z in zone_of])
    drv = res_aos(nxt["drv_cpu"], nxt["drv_mem"], nxt["drv_gpu"]); exe = res_aos(nxt["exe_cpu"], nxt["exe_mem"], nxt["exe_gpu"])
    wd, we, woff = cl.binpack_batch(2, drv, exe, nxt["count"], [names[i] for i in order], [names[i] for i in order], with_efficiencies=True)
    assert np.array_equal(gd, wd)
    for i in np.nonzero(wd >= 0)[0]:
        assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]])


def test_refusals(packer, gangpack):
    import torch
    zones, eo, do, eoff, doff = az_layout(ORDER_D8, ORDER_E8, ZONE8)
    Z = len(zones)
    apps = _apps([(1000, G, 1000, G, 2)])
    n = len(CPU8)
    gpu = np.zeros(n, np.int64)

    def fresh():
        packer.set_snapshot(CPU8, MEM8, gpu, eo, do, eoff, doff)
        packer.set_schedulable(CPU8, MEM8, gpu)

    def refused(match, mode=1, e=ORDER_E8, d=ORDER_D8, z=Z):
        with pytest.raises(gangpack.native.GangpackError) as ei:
            packer.pack_fifo_az_aware(apps, mode, e, d, z)
        assert ei.value.status == 1 and match in str(ei.value), str(ei.value)

    fresh()
    packer.pack_fifo_az_aware(apps, 1, ORDER_E8, ORDER_D8, Z)           # the well-formed call goes through
    fresh(); refused("FIFO modes", mode=0)
    fresh(); refused("0..64", z=65)
    fresh(); refused("exceeds the snapshot's instance groups", z=len(eoff))
    packer.set_snapshot(CPU8, MEM8, gpu, eo, do, eoff, doff); refused("gp_set_schedulable first")
    fresh(); refused("exec_order entry out of range", e=ORDER_E8[:-1] + [n])
    fresh(); refused("drv_order lists a node twice", d=ORDER_D8[:-1] + [ORDER_D8[0]])
    fresh(); refused("does not list as an executor candidate", e=ORDER_E8[:-1] + [2])          # node 2: driver only
    fresh(); refused("does not list as a driver candidate", d=ORDER_D8[:-1] + [3])             # node 3: executor only
    fresh(); refused("order lengths", e=ORDER_E8[:-1])
    moved = [0, 3, 4, 1, 6, 5, 7]                                       # every zone keeps its relative order: accepted
    fresh(); packer.pack_fifo_az_aware(apps, 1, moved, ORDER_D8, Z)
    fresh(); refused("zone group 0's executor order", e=[3, 1, 4, 0, 6, 5, 7])
    fresh(); refused("zone group 1's driver order", d=[2, 0, 7, 1, 6])
    t = lambda a, dt: torch.as_tensor(np.asarray(a), dtype=dt, device="cuda")
    keep = [t(CPU8, torch.int64), t(MEM8, torch.int64), t(gpu, torch.int64), t(eoff, torch.int32), t(eo, torch.int32),
            t(doff, torch.int32), t(do, torch.int32)]
    packer.set_snapshot_device(*keep)
    packer.set_schedulable(CPU8, MEM8, gpu)
    refused("laid out by gp_set_snapshot")
    packer.synchronize()
