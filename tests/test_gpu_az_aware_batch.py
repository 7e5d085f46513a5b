"""gp_pack_batch_az_aware = AzAwareTightlyPack (az_aware_pack_tightly.go:27-38) for a batch of independent decisions in one
call: every application is packed in every candidate zone with tightly-pack and chosen by packing efficiency like
gp_pack_batch_zones, and when no zone wins SparkBinPack(tightlyPackExecutors) runs over the undivided orders, on the
device, against the unmodified snapshot.

Every case checks the call against
- the literal restatement (orc_binpack_batch with the az-aware packer over the undivided name orders): every driver_node
  and the ExecutorNodes of every placed application;
- the two-context recipe it replaces (gp_pack_batch_zones on a zone-only snapshot, then gp_pack_batch over the undivided
  orders for the zone -1 applications): zone, driver_node and slices equal, avg_efficiency bit-identical for zone winners
  and zero for the rest;
- gp_stats.scan_path_apps == the number of zone -1 applications, and the snapshot left as it was.
Cases under 400 nodes also walk the batch in pure Python (pyref) for the zone / fallback split."""
import numpy as np
import pytest

from helpers import node_names, random_apps, random_cluster, res_aos
from oracle import pyref

pytestmark = pytest.mark.gpu

ORC_AZ_AWARE = 3
G = 1 << 30


def az_layout(order_d, order_e, zone_of):
    """The snapshot layout of az-aware-tightly-pack: one group per candidate zone (driverZonesInOrder order, zones without
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


APP_KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")


def az_two_context_recipe(packer_z, packer_u, cpu, mem, gpu, sched, layout, order_e, order_d, apps):
    """Independent az-aware-tightly-pack as two calls on two contexts: gp_pack_batch_zones on a snapshot of the candidate
    zones alone (packer_z), then, for the applications no zone won, gp_pack_batch(tightly-pack, independent) over the
    undivided orders on the second context (packer_u).  -> (zone, driver_node, executor_nodes, off, avg_efficiency)."""
    zones, eo, do, eoff, doff = layout
    Z = len(zones)
    q = len(apps["count"])
    off = np.zeros(q + 1, np.int64)
    np.cumsum(np.maximum(np.asarray(apps["count"], np.int64), 0), out=off[1:])
    if Z:
        packer_z.set_snapshot(cpu, mem, gpu, eo[:eoff[Z]], do[:doff[Z]], eoff[:Z + 1], doff[:Z + 1])
        packer_z.set_schedulable(*sched)
        zone, drv, exe, _, avg = packer_z.pack_batch_zones(apps, 0)
        drv, exe = drv.copy(), exe.copy()
    else:
        zone, drv = np.full(q, -1, np.int32), np.full(q, -1, np.int32)
        exe, avg = np.full(int(off[-1]), -9, np.int32), np.zeros((q, 4))
    fb = np.nonzero(zone == -1)[0]
    if fb.size:
        packer_u.set_snapshot(cpu, mem, gpu, order_e, order_d)
        sub = {k: np.asarray(apps[k])[fb] for k in APP_KEYS}
        d2, e2, o2 = packer_u.pack_batch(sub, 0, 0)
        drv[fb] = d2
        for j in np.nonzero(d2 >= 0)[0]:
            i = fb[j]
            exe[off[i]:off[i + 1]] = e2[o2[j]:o2[j + 1]]
    return zone, drv, exe, off, avg


@pytest.fixture(scope="module")
def packers(gangpack):
    ps = [gangpack.GangPacker() for _ in range(3)]         # the call under test, and the two contexts of the recipe
    yield ps
    for p in ps:
        p.close()


def run_case(oracle, packers, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, label, walk=True, literal=True):
    """-> (zone, driver_node, executor_nodes, off, avg, stats) of gp_pack_batch_az_aware after every check."""
    p, pz, pu = packers
    n = len(cpu)
    layout = az_layout(order_d, order_e, zone_of)
    zones, eo, do, eoff, doff = layout
    p.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    p.set_schedulable(sc, sm, sg)
    zone, gd, ge, goff, avg = p.pack_batch_az_aware(apps, order_e, order_d, len(zones))
    st = p.stats()
    for x, y in zip(p.get_snapshot(), (cpu, mem, gpu)):                 # independent decisions: nothing is charged
        assert np.array_equal(x, y), label
    assert st["scan_path_apps"] == int((zone == -1).sum()), (label, st)
    assert ((zone >= -1) & (zone < max(len(zones), 1))).all() and (gd >= -1).all(), label
    assert (gd[zone >= 0] >= 0).all(), label
    # the two-context recipe
    rz, rd, re, roff, ravg = az_two_context_recipe(pz, pu, cpu, mem, gpu, (sc, sm, sg), layout, order_e, order_d, apps)
    assert np.array_equal(goff, roff)
    assert np.array_equal(zone, rz), (label, np.nonzero(zone != rz)[0][:5])
    assert np.array_equal(gd, rd), (label, np.nonzero(gd != rd)[0][:5])
    placed = np.zeros(int(goff[-1]), bool)
    for i in np.nonzero(gd >= 0)[0]:
        placed[goff[i]:goff[i + 1]] = True
    assert np.array_equal(ge[placed], re[placed]), label
    won = zone >= 0
    assert np.array_equal(avg[won].view(np.uint64), ravg[won].view(np.uint64)), label      # bit for bit
    assert (avg[~won] == 0.0).all(), label
    # the literal restatement
    if literal:
        names = node_names(n)
        cl = oracle.Cluster(names, cpu, mem, gpu, sched=(sc, sm, sg), zone=["zone-%d" % z for z in zone_of])
        drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"]); exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
        wd, we, woff = cl.binpack_batch(ORC_AZ_AWARE, drv, exe, apps["count"], [names[i] for i in order_d], [names[i] for i in order_e],
                                        with_efficiencies=True, n_threads=8)
        assert np.array_equal(goff, woff)
        bad = np.nonzero(gd != wd)[0]
        assert bad.size == 0, (label, bad[:5], gd[bad[:5]], wd[bad[:5]], zone[bad[:5]])
        assert np.array_equal(ge[placed], we[placed]), label
        if walk and n < 400:
            _walk(names, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, zones, apps, zone, gd, ge, goff, label)
    return zone, gd, ge, goff, avg, st


def _walk(names, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, zones, apps, zone, gd, ge, goff, label):
    """pyref: zone[i] is the winner of single_az_tightly_pack, or -1 and az_aware_tightly_pack's fallback placement."""
    meta = {names[i]: (int(cpu[i]), int(mem[i]), int(gpu[i])) for i in range(len(names))}
    sched = {names[i]: (int(sc[i]), int(sm[i]), int(sg[i])) for i in range(len(names))}
    zmap = {names[i]: "zone-%d" % zone_of[i] for i in range(len(names))}
    zlabels = ["zone-%d" % z for z in zones]
    dnames = [names[i] for i in order_d]; enames = [names[i] for i in order_e]
    for i in range(len(apps["count"])):
        d_req = (int(apps["drv_cpu"][i]), int(apps["drv_mem"][i]), int(apps["drv_gpu"][i]))
        e_req = (int(apps["exe_cpu"][i]), int(apps["exe_mem"][i]), int(apps["exe_gpu"][i]))
        k = int(apps["count"][i])
        d, ex, ok = pyref.single_az_tightly_pack(d_req, e_req, k, dnames, enames, meta, sched, zmap)
        if ok:
            assert zone[i] == zlabels.index(zmap[d]), (label, i)
        else:
            assert zone[i] == -1, (label, i)
            d, ex, ok = pyref.az_aware_tightly_pack(d_req, e_req, k, dnames, enames, meta, sched, zmap)
        assert ok == (gd[i] >= 0), (label, i)
        if ok:
            assert names[gd[i]] == d and [names[j] for j in ge[goff[i]:goff[i + 1]]] == ex, (label, i)


def _random_case(seed):
    rng = np.random.default_rng(9900 + seed)
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
    apps["count"] = np.where(big, rng.integers(20, 300, q), apps["count"]).astype(np.int32)
    return cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps


@pytest.mark.parametrize("seed", range(6))
def test_az_aware_batch_randomized(oracle, packers, seed):
    *_, st = run_case(oracle, packers, *_random_case(seed), label=f"seed {seed}")
    assert st["scan_path_apps"] > 0, seed


def _apps(rows):
    """rows: (drv_cpu, drv_mem, exe_cpu, exe_mem, count)"""
    r = np.array(rows, np.int64).reshape(-1, 5)
    q = len(r)
    return {"drv_cpu": r[:, 0], "drv_mem": r[:, 1], "drv_gpu": np.zeros(q, np.int64), "exe_cpu": r[:, 2], "exe_mem": r[:, 3],
            "exe_gpu": np.zeros(q, np.int64), "count": r[:, 4].astype(np.int32)}


# zone 0: nodes 0-1 (driver + executor candidates); zone 1: node 2, driver candidate only; zone 2: nodes 3-5, executor
# candidates only; zone 3: nodes 6-7 (driver + executor candidates, the second candidate zone)
CPU8 = np.array([4000, 4000, 12000, 4000, 4000, 4000, 4000, 4000], np.int64)
MEM8 = np.full(8, 64 * G, np.int64)
ZONE8 = np.array([0, 0, 1, 2, 2, 2, 3, 3])
ORDER_E8 = [3, 0, 4, 1, 6, 5, 7]
ORDER_D8 = [2, 0, 6, 1, 7]


def _constructed(oracle, packers, apps, label, cpu=CPU8, mem=MEM8, sc=None, sm=None, literal=True):
    n = len(cpu)
    sc = cpu + 4000 if sc is None else sc
    sm = mem + 8 * G if sm is None else sm
    return run_case(oracle, packers, cpu, mem, np.zeros(n, np.int64), sc, sm, np.zeros(n, np.int64),
                    ZONE8, ORDER_D8, ORDER_E8, apps, label, literal=literal)


def test_fallback_spans_the_trailing_group(oracle, packers):
    """The driver only fits on the driver-only zone's node and its executors land on the executor-only zone's nodes and
    zone 0's, in the undivided order: only the trailing group reaches those nodes.  exe_count 0 takes the same path; the
    third application fits in a zone."""
    apps = _apps([(6000, G, 2000, G, 6), (5000, G, 1000, G, 0), (1000, G, 1000, G, 2)])
    zone, gd, ge, goff, avg, st = _constructed(oracle, packers, apps, "trailing group")
    assert list(zone) == [-1, -1, 0] and list(gd[:2]) == [2, 2] and st["scan_path_apps"] == 2
    assert list(ge[goff[0]:goff[1]]) == [3, 3, 0, 0, 4, 4]
    assert avg[2, 3] > 0.0


def test_every_and_no_application_falls_back(oracle, packers):
    every = _apps([(6000, G, 1000 * (1 + i % 3), G, i % 5) for i in range(40)])
    zone, gd, *_, st = _constructed(oracle, packers, every, "every")
    assert (zone == -1).all() and (gd == 2).all() and st["scan_path_apps"] == 40
    none = _apps([(500 * (i % 3), G, 250 * (1 + i % 4), G, i % 4) for i in range(40)])
    zone, gd, *_, st = _constructed(oracle, packers, none, "none")
    assert (zone >= 0).all() and st["scan_path_apps"] == 0


def test_one_application(oracle, packers):
    """The Predicate's own pack: one decision, zone winner and fallback."""
    for rows, want_zone in (([(1000, G, 1000, G, 3)], 0), ([(6000, G, 1000, G, 3)], -1), ([(6000, G, 9000, G, 3)], -1)):
        zone, gd, *_ = _constructed(oracle, packers, _apps(rows), f"one {rows}")
        assert zone[0] == want_zone
    assert gd[0] == -1                                                  # the last one fits nowhere


def test_no_candidate_zone_is_independent_tightly_pack(oracle, packers):
    """n_zones = 0: every application takes the fallback, which is then gp_pack_batch(tightly-pack, independent) on the
    undivided one-group snapshot."""
    rng = np.random.default_rng(606)
    n = 120
    cpu, mem, gpu = random_cluster(rng, n)
    zone_of = np.where(np.arange(n) % 2 == 0, 0, 1)
    order_e = [int(i) for i in rng.permutation(n) if zone_of[i] == 0]
    order_d = [int(i) for i in rng.permutation(n) if zone_of[i] == 1]
    apps = random_apps(rng, 200)
    zone, gd, ge, goff, _, st = run_case(oracle, packers, cpu, mem, gpu, cpu + 1000, mem + G, gpu, zone_of, order_d, order_e, apps,
                                         "no zones")
    assert (zone == -1).all() and st["scan_path_apps"] == 200 and (gd >= 0).any()
    p = packers[1]
    p.set_snapshot(cpu, mem, gpu, order_e, order_d)
    bd, be, boff = p.pack_batch(apps, 0, 0)
    assert np.array_equal(bd, gd)
    for i in np.nonzero(gd >= 0)[0]:
        assert np.array_equal(be[boff[i]:boff[i + 1]], ge[goff[i]:goff[i + 1]])


@pytest.mark.parametrize("Z", [64, 65, 70, 100])
def test_many_zones_and_a_trailing_group(oracle, packers, Z):
    """No 64-zone bound: Z candidate zones plus a driver-only and an executor-only zone in the trailing group."""
    rng = np.random.default_rng(6400 + Z)
    per = 3
    n = (Z + 2) * per
    cpu, mem, gpu = random_cluster(rng, n)
    sc, sm = cpu + rng.integers(0, 9, n) * 250, mem + rng.integers(0, 17, n) * (1 << 28)
    zone_of = rng.permutation(np.arange(n) % (Z + 2))
    order_e = [int(i) for i in rng.permutation(n) if zone_of[i] != Z]              # zone Z: driver candidates only
    order_d = [int(i) for i in rng.permutation(n) if zone_of[i] != Z + 1]          # zone Z + 1: executor candidates only
    apps = random_apps(rng, 150)
    apps["count"] = np.where(rng.random(150) < 0.2, rng.integers(10, 40, 150), apps["count"]).astype(np.int32)
    assert len(az_layout(order_d, order_e, zone_of)[0]) == Z
    zone, gd, *_, st = run_case(oracle, packers, cpu, mem, gpu, sc, sm, gpu.clip(0), zone_of, order_d, order_e, apps, f"{Z} zones")
    assert (zone >= 16).any() and st["scan_path_apps"] > 0


def test_ties_and_zero_efficiency(oracle, packers):
    """Zones 0 and 3 are identical: every tie goes to the first zone.  A driver-only application with zero requests on
    untouched nodes has an average efficiency of exactly 0.0 in every zone, so no zone wins and the fallback places it."""
    cpu = np.full(8, 8000, np.int64)
    apps = _apps([(1000, G, 1000, G, 2), (0, 0, 1000, G, 0), (500, G, 2000, 2 * G, 1)])
    zone, gd, _, _, avg, st = _constructed(oracle, packers, apps, "ties", cpu=cpu, sc=cpu, sm=MEM8)
    assert zone[0] == 0 and zone[2] == 0
    assert zone[1] == -1 and gd[1] >= 0 and (avg[1] == 0.0).all() and st["scan_path_apps"] == 1


def test_general_class_and_negative_gpu(oracle, packers):
    """Requests and availabilities of 2^32 and more (the general arithmetic class) and negative gpu availabilities."""
    rng = np.random.default_rng(78)
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
    *_, st = run_case(oracle, packers, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, "general class")
    assert st["scan_path_apps"] > 0


def _count_cluster(count):
    """ZONE8 with one executor per milli-core: each candidate zone holds about count / 2, the executor candidates together
    about 7 / 4 count."""
    cap = count // 4 + 1
    cpu = np.full(8, cap, np.int64)
    cpu[2] = cap + 1000                                                 # the driver-only node
    return cpu, np.full(8, 1 << 40, np.int64)


@pytest.mark.parametrize("count", [65535, 65536, (1 << 20) + 1, 1 << 24])
def test_large_fallback_counts(oracle, packers, count):
    """Counts no zone holds, placed by the fallback; 2^20 (the FIFO bound) and above against the recipe and the closed form."""
    cpu, mem = _count_cluster(count)
    apps = _apps([(500, 1, 1, 1, count), (500, 1, 1, 1, 3)])
    literal = count < (1 << 20)
    zone, gd, ge, goff, _, _ = _constructed(oracle, packers, apps, f"count {count}", cpu=cpu, mem=mem, literal=literal)
    assert zone[0] == -1 and gd[0] >= 0 and zone[1] >= 0
    if not literal:
        one = {k: apps[k][:1] for k in APP_KEYS}
        _, wd, we, _, _ = oracle.closed_batch(0, 0, cpu, mem, np.zeros(8, np.int64), np.array(ORDER_D8, np.int32),
                                              np.array(ORDER_E8, np.int32), res_aos(one["drv_cpu"], one["drv_mem"], one["drv_gpu"]),
                                              res_aos(one["exe_cpu"], one["exe_mem"], one["exe_gpu"]), one["count"])
        assert wd[0] == gd[0] and np.array_equal(we[:count], ge[goff[0]:goff[1]])


def test_count_above_2_24_is_refused(packers, gangpack):
    count = (1 << 24) + 1
    cpu, mem = _count_cluster(count)
    zones, eo, do, eoff, doff = az_layout(ORDER_D8, ORDER_E8, ZONE8)
    p = packers[0]
    p.set_snapshot(cpu, mem, np.zeros(8, np.int64), eo, do, eoff, doff)
    p.set_schedulable(cpu, mem, np.zeros(8, np.int64))
    with pytest.raises(gangpack.native.GangpackError) as ei:
        p.pack_batch_az_aware(_apps([(500, 1, 1, 1, count)]), ORDER_E8, ORDER_D8, len(zones))
    assert ei.value.status == 6


def test_one_context_across_entry_points(packers, gangpack):
    """gp_pack_batch_az_aware, gp_pack_fifo_az_aware, gp_pack_batch_az_aware on one context give what each gives on a fresh
    context holding the same snapshot."""
    cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps = _random_case(3)
    zones, eo, do, eoff, doff = az_layout(order_d, order_e, zone_of)
    Z = len(zones)
    fifo_apps = dict(apps, young=np.ones(len(apps["count"]), np.uint8))

    def fresh(avail):
        f = gangpack.GangPacker()
        f.set_snapshot(*avail, eo, do, eoff, doff)
        f.set_schedulable(sc, sm, sg)
        return f

    p = packers[0]
    p.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    p.set_schedulable(sc, sm, sg)
    got = [p.pack_batch_az_aware(apps, order_e, order_d, Z)]
    got.append(p.pack_fifo_az_aware(fifo_apps, 2, order_e, order_d, Z))
    charged = p.get_snapshot()
    got.append(p.pack_batch_az_aware(apps, order_e, order_d, Z))
    want = []
    for avail, call in (((cpu, mem, gpu), lambda f: f.pack_batch_az_aware(apps, order_e, order_d, Z)),
                        ((cpu, mem, gpu), lambda f: f.pack_fifo_az_aware(fifo_apps, 2, order_e, order_d, Z)),
                        (charged, lambda f: f.pack_batch_az_aware(apps, order_e, order_d, Z))):
        f = fresh(avail)
        try:
            want.append(call(f))
        finally:
            f.close()
    for k, (g_, w_) in enumerate(zip(got, want)):
        zone, gd, ge, goff, avg = g_
        assert np.array_equal(zone, w_[0]) and np.array_equal(gd, w_[1]) and np.array_equal(avg, w_[4]), k
        for i in np.nonzero(gd >= 0)[0]:
            assert np.array_equal(ge[goff[i]:goff[i + 1]], w_[2][goff[i]:goff[i + 1]]), (k, i)
    assert not np.array_equal(got[0][1], got[2][1])                     # the FIFO loop's charges changed the decisions


def test_refusals(packers, gangpack):
    import torch
    zones, eo, do, eoff, doff = az_layout(ORDER_D8, ORDER_E8, ZONE8)
    Z = len(zones)
    apps = _apps([(1000, G, 1000, G, 2)])
    n = len(CPU8)
    gpu = np.zeros(n, np.int64)
    p = packers[0]

    def fresh():
        p.set_snapshot(CPU8, MEM8, gpu, eo, do, eoff, doff)
        p.set_schedulable(CPU8, MEM8, gpu)

    def refused(match, e=ORDER_E8, d=ORDER_D8, z=Z):
        with pytest.raises(gangpack.native.GangpackError) as ei:
            p.pack_batch_az_aware(apps, e, d, z)
        assert ei.value.status == 1 and match in str(ei.value), str(ei.value)

    fresh()
    p.pack_batch_az_aware(apps, ORDER_E8, ORDER_D8, Z)                   # the well-formed call goes through
    fresh(); p.pack_batch_az_aware(apps, ORDER_E8, ORDER_D8, len(eoff) - 1)     # every group a zone: accepted
    fresh(); refused("n_zones is negative", z=-1)
    fresh(); refused("exceeds the snapshot's instance groups", z=len(eoff))
    p.set_snapshot(CPU8, MEM8, gpu, eo, do, eoff, doff); refused("gp_set_schedulable first")
    fresh(); refused("exec_order entry out of range", e=ORDER_E8[:-1] + [n])
    fresh(); refused("drv_order entry out of range", d=ORDER_D8[:-1] + [-1])
    fresh(); refused("exec_order lists a node twice", e=ORDER_E8[:-1] + [ORDER_E8[0]])
    fresh(); refused("drv_order lists a node twice", d=ORDER_D8[:-1] + [ORDER_D8[0]])
    fresh(); refused("does not list as an executor candidate", e=ORDER_E8[:-1] + [2])          # node 2: driver only
    fresh(); refused("does not list as a driver candidate", d=ORDER_D8[:-1] + [3])             # node 3: executor only
    fresh(); refused("order lengths", e=ORDER_E8[:-1])
    fresh(); refused("order lengths", d=ORDER_D8 + [3])
    fresh(); refused("zone group 0's executor order", e=[3, 1, 4, 0, 6, 5, 7])
    fresh(); refused("zone group 1's driver order", d=[2, 0, 7, 1, 6])
    t = lambda a, dt: torch.as_tensor(np.asarray(a), dtype=dt, device="cuda")
    keep = [t(CPU8, torch.int64), t(MEM8, torch.int64), t(gpu, torch.int64), t(eoff, torch.int32), t(eo, torch.int32),
            t(doff, torch.int32), t(do, torch.int32)]
    p.set_snapshot_device(*keep)
    p.set_schedulable(CPU8, MEM8, gpu)
    refused("laid out by gp_set_snapshot")
    p.synchronize()


def test_full_size(oracle, packers):
    """10 000 nodes in 8 zones of unequal size, 100 000 synth applications, every 100th larger than the largest zone holds:
    all decisions against the recipe, the first 3 000 (30 of them large) against the literal restatement."""
    from k8s_spark_scheduler_b200 import synth
    n, q, Z = 10000, 100000, 8
    nodes = synth.make_nodes(n)
    cpu, mem, gpu = nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"]
    sc, sm, sg = nodes["alloc_cpu"], nodes["alloc_mem"], nodes["alloc_gpu"]
    order = [int(i) for i in synth.priority_order(cpu, mem)]
    share = np.array([0.3, 0.2, 0.15, 0.1, 0.1, 0.07, 0.05, 0.03])
    zone_of = np.searchsorted(np.cumsum(share), (np.arange(n) * 0.6180339887) % 1.0, side="right").clip(0, Z - 1)
    s = synth.make_apps(q, seed=21)
    apps = {k: np.array(s[k]) for k in APP_KEYS}
    for i in range(0, q, 100):
        caps = np.minimum(np.maximum(cpu, 0) // int(apps["exe_cpu"][i]), np.maximum(mem, 0) // int(apps["exe_mem"][i]))
        apps["count"][i] = int(max(caps[zone_of == z].sum() for z in range(Z))) + 1 + i % 7
    zone, gd, ge, goff, avg, st = run_case(oracle, packers, cpu, mem, gpu, sc, sm, sg, zone_of, order, order, apps, "full size",
                                           literal=False)
    assert st["scan_path_apps"] >= q // 100 and ((zone == -1) & (gd >= 0)).any()
    sel = np.arange(3000)
    sub = {k: apps[k][sel] for k in APP_KEYS}
    names = node_names(n)
    cl = oracle.Cluster(names, cpu, mem, gpu, sched=(sc, sm, sg), zone=["zone-%d" % z for z in zone_of])
    drv = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"]); exe = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
    onames = [names[i] for i in order]
    wd, we, woff = cl.binpack_batch(ORC_AZ_AWARE, drv, exe, sub["count"], onames, onames, with_efficiencies=True, n_threads=8)
    assert np.array_equal(gd[sel], wd)
    for j, i in enumerate(sel):
        if wd[j] >= 0:
            assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[j]:woff[j + 1]]), i
