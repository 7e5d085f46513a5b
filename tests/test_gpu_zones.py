"""SURVEY 8f row f3 on the device: single-az-tightly-pack / single-az-minimal-fragmentation for a batch
(gp_pack_batch_zones: pack every zone, float64 packing efficiencies and chooseBestResult in a kernel) against the LITERAL
restatement of getSingleAZSparkBinFunction + chooseBestResult + ComputePackingEfficiencies (LIB/binpack/single_az.go:23-97,
efficiency.go:66-156) -- the choice must be bit-identical: same zone, same driver node, same ExecutorNodes."""
import numpy as np
import pytest

from helpers import node_names, random_apps, random_cluster, res_aos

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def _zone_groups(order_d, order_e, zone_of):
    """groupNodesByZone (single_az.go:57-73) for both orders; zones without executor candidates are skipped (:38-41)."""
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
    return zones, np.array(eo, np.int32), np.array(do, np.int32), np.array(eoff, np.int32), np.array(doff, np.int32)


@pytest.mark.parametrize("seed", range(8))
def test_single_az_packers_vs_literal(oracle, packer, seed):
    rng = np.random.default_rng(700 + seed)
    n = int(rng.integers(30, 160))
    Z = int(rng.integers(1, 5))
    cpu, mem, gpu = random_cluster(rng, n, tight=bool(seed % 2), gpus=bool(seed % 3 == 0))
    # schedulable = available + what is already used (whole cores and odd millicores both occur: Value() rounds up)
    sc = cpu + rng.integers(0, 9, n) * 250 + (rng.integers(0, 3, n) == 0) * 1
    sm = mem + rng.integers(0, 17, n) * (1 << 28)
    sg = np.maximum(gpu, 0) + (rng.integers(0, 2, n) if seed % 3 == 0 else 0)
    zone_of = rng.integers(0, Z, n)
    names = node_names(n)
    labels = ["zone-%d" % z for z in zone_of]
    order = rng.permutation(n)
    order_e = [int(i) for i in order if rng.random() < 0.85]
    order_d = [int(i) for i in rng.permutation(n)[: max(1, int(n * 0.7))]]
    zones, eo, do, eoff, doff = _zone_groups(order_d, order_e, zone_of)
    q = 250
    apps = random_apps(rng, q, gpus=bool(seed % 3 == 0), zero_dims=bool(seed == 5))
    cl = oracle.Cluster(names, cpu, mem, gpu, sched=(sc, sm, sg), zone=labels)
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"]); exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    if not zones:
        return
    packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    packer.set_schedulable(sc, sm, sg)
    for algo, oalgo in ((0, 2), (2, 5)):                       # single-az-tightly-pack, single-az-minimal-fragmentation
        wd, we, woff = cl.binpack_batch(oalgo, drv, exe, apps["count"], [names[i] for i in order_d], [names[i] for i in order_e],
                                        with_efficiencies=True, n_threads=4)
        zone, gd, ge, goff, avg = packer.pack_batch_zones(apps, algo)
        assert np.array_equal(goff, woff)
        bad = np.nonzero(gd != wd)[0]
        assert bad.size == 0, (seed, algo, bad[:5], gd[bad[:5]], wd[bad[:5]])
        for i in np.nonzero(wd >= 0)[0]:
            assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]]), (seed, algo, i)
            assert zone[i] == zones.index(zone_of[wd[i]])
            assert avg[i, 3] > 0.0
        assert (zone[wd < 0] == -1).all()


def _fifo_zone_case(rng, seed, n, Z, q, tight):
    cpu, mem, gpu = random_cluster(rng, n, tight=tight, gpus=bool(seed % 3 == 0))
    sc = cpu + rng.integers(0, 9, n) * 250 + (rng.integers(0, 3, n) == 0) * 1
    sm = mem + rng.integers(0, 17, n) * (1 << 28)
    sg = np.maximum(gpu, 0) + (rng.integers(0, 2, n) if seed % 3 == 0 else 0)
    zone_of = rng.integers(0, Z, n)
    order_e = [int(i) for i in rng.permutation(n) if rng.random() < 0.9]
    order_d = [int(i) for i in rng.permutation(n)[: max(1, int(n * 0.7))]]
    apps = random_apps(rng, q, gpus=bool(seed % 3 == 0), zero_dims=bool(seed == 5))
    apps["young"] = (rng.random(q) < (0.97 if seed % 2 else 1.0)).astype(np.uint8)      # odd seeds: the queue may block
    return cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps


@pytest.mark.parametrize("seed", range(6))
def test_fifo_with_single_az_packers_vs_literal(oracle, packer, seed):
    """gp_pack_fifo_zones = fitEarlierDrivers (resource.go:224-262) with SingleAZTightlyPack / SingleAZMinimalFragmentation as
    BinpackFunc, one launch for the whole queue: zone choice, placements, blocking and the availability left behind must equal
    the literal restatement's loop (which packs every zone, compares the float64 averages and subtracts the winner's usage
    per driver), in both accounting modes."""
    rng = np.random.default_rng(4100 + seed)
    n = int(rng.integers(40, 200)); Z = int(rng.integers(1, 6)); q = 220
    cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps = _fifo_zone_case(rng, seed, n, Z, q, tight=bool(seed % 2))
    names = node_names(n)
    labels = ["zone-%d" % z for z in zone_of]
    zones, eo, do, eoff, doff = _zone_groups(order_d, order_e, zone_of)
    if not zones:
        return
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"]); exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    for algo, oalgo in ((0, 2), (2, 5)):
        for mode in (1, 2):
            cl = oracle.Cluster(names, cpu, mem, gpu, sched=(sc, sm, sg), zone=labels)
            blocked, wd, we, woff = cl.fifo(oalgo, mode, drv, exe, apps["count"], apps["young"], [names[i] for i in order_d],
                                            [names[i] for i in order_e], with_efficiencies=True)
            packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
            packer.set_schedulable(sc, sm, sg)
            zone, gd, ge, goff, avg = packer.pack_fifo_zones(apps, algo, mode)
            assert np.array_equal(goff, woff)
            bad = np.nonzero(gd != wd)[0]
            assert bad.size == 0, (seed, algo, mode, bad[:5], gd[bad[:5]], wd[bad[:5]], blocked)
            for i in np.nonzero(wd >= 0)[0]:
                assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]]), (seed, algo, mode, i)
                assert zone[i] == zones.index(zone_of[wd[i]])
            assert (zone[wd < 0] == -1).all()
            fc, fm, fg = packer.get_snapshot()
            wc, wm, wg = cl.available()
            assert np.array_equal(fc, wc) and np.array_equal(fm, wm) and np.array_equal(fg, wg), (seed, algo, mode)
    # the device keeps the availability the loop left: an independent zone batch right after sees it
    zone2, gd2, ge2, goff2, _ = packer.pack_batch_zones(apps, 0)
    wd2, we2, woff2 = cl.binpack_batch(2, drv, exe, apps["count"], [names[i] for i in order_d], [names[i] for i in order_e], with_efficiencies=True)
    # (cl holds the state of the last loop: minimal-fragmentation, exact accounting -- the same the device just ran)
    assert np.array_equal(gd2, wd2)


def test_fifo_zones_blocks_and_rejects(oracle, packer, gangpack):
    """A driver that fits in no zone and is not young stops the queue (-2 behind it, resource.go:244-253); wrong modes /
    packers are refused."""
    n = 12
    cpu = np.full(n, 8000, np.int64); mem = np.full(n, 32 << 30, np.int64); gpu = np.zeros(n, np.int64)
    zone_of = np.arange(n) % 3
    order = list(range(n))
    zones, eo, do, eoff, doff = _zone_groups(order, order, zone_of)
    packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    packer.set_schedulable(cpu, mem, gpu)
    apps = {"drv_cpu": np.array([1000, 1000, 1000, 1000], np.int64), "drv_mem": np.full(4, 1 << 30, np.int64), "drv_gpu": np.zeros(4, np.int64),
            "exe_cpu": np.array([2000, 4000, 2000, 2000], np.int64), "exe_mem": np.full(4, 2 << 30, np.int64), "exe_gpu": np.zeros(4, np.int64),
            "count": np.array([3, 40, 2, 2], np.int32), "young": np.array([0, 1, 0, 0], np.uint8)}
    zone, gd, ge, goff, _ = packer.pack_fifo_zones(apps, 0, 1)
    assert gd[0] >= 0 and gd[1] == -1 and gd[2] >= 0 and gd[3] >= 0          # the young driver is skipped
    apps["young"][1] = 0
    packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    packer.set_schedulable(cpu, mem, gpu)                                      # a new snapshot drops the schedulable resources
    zone, gd, ge, goff, _ = packer.pack_fifo_zones(apps, 0, 1)
    assert gd[0] >= 0 and list(gd[1:]) == [-1, -2, -2] and list(zone[1:]) == [-1, -1, -1]
    with pytest.raises(gangpack.native.GangpackError):
        packer.pack_fifo_zones(apps, 1, 1)                                      # distribute-evenly has no single-AZ form
    with pytest.raises(gangpack.native.GangpackError):
        packer.pack_fifo_zones(apps, 0, 0)                                      # independent decisions: gp_pack_batch_zones


def test_zones_after_fifo_sees_charged_availability(oracle, packer):
    """The efficiencies read the availability the FIFO batch left behind (node-table copy refreshed from the slots)."""
    rng = np.random.default_rng(9)
    n = 60
    cpu = (rng.integers(8, 32, n) * 1000).astype(np.int64); mem = (rng.integers(16, 64, n) << 30).astype(np.int64); gpu = np.zeros(n, np.int64)
    sc, sm, sg = cpu + 4000, mem + (8 << 30), gpu
    zone_of = np.arange(n) % 3
    names = node_names(n)
    order = [int(i) for i in np.lexsort((np.arange(n), cpu, mem))]
    zones, eo, do, eoff, doff = _zone_groups(order, order, zone_of)
    queue = random_apps(rng, 40); queue["group"] = (np.arange(40) % len(zones)).astype(np.int32); queue["young"] = np.ones(40, np.uint8)
    packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    packer.pack_batch(queue, 0, 2)
    fc, fm, fg = packer.get_snapshot()
    assert not np.array_equal(fc, cpu)
    packer.set_schedulable(sc, sm, sg)
    mine = random_apps(rng, 60)
    zone, gd, ge, goff, _ = packer.pack_batch_zones(mine, 0)
    cl = oracle.Cluster(names, fc, fm, fg, sched=(sc, sm, sg), zone=["zone-%d" % z for z in zone_of])
    drv = res_aos(mine["drv_cpu"], mine["drv_mem"], mine["drv_gpu"]); exe = res_aos(mine["exe_cpu"], mine["exe_mem"], mine["exe_gpu"])
    wd, we, woff = cl.binpack_batch(2, drv, exe, mine["count"], [names[i] for i in order], [names[i] for i in order], with_efficiencies=True)
    assert np.array_equal(gd, wd)
    for i in np.nonzero(wd >= 0)[0]:
        assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]])


def test_reservation_table_and_resident_snapshot(oracle, packer):
    """gp_reserve_placements = newResourceReservation (resourcereservations.go:491-528) for a batch + exact charging of the
    device-resident snapshot; gp_apply_usage_delta releases / adds reservations.  Rows: slot 0 = "driver" on DriverNode with
    the driver's resources, slot i = "executor-i" on ExecutorNodes[i-1] with the executor's resources.  The availability
    the device then holds equals allocatable - UsageForNodes(reservations) (resources.go:31-43), and a following batch packs
    against it like the oracle does on the recomputed availability."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(800)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    drv_order = order[: 500]                                   # some executor candidates are no driver candidates ...
    exe_order = order[100:]                                    # ... and vice versa (spare driver slots)
    apps = synth.make_apps(300, seed=3)
    KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
    a = {k: apps[k] for k in KEYS}
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], exe_order, drv_order)
    placed = packer.pack_batch(a, 0, 0)
    # independent decisions may overcommit a node between them: reserving all of them is still well defined (negative availability)
    rows = packer.reserve_placements(a, placed, subtract=True)
    dn, en, off = placed
    exp = []
    for i in range(300):
        if dn[i] < 0:
            continue
        exp.append((i, 0, dn[i], a["drv_cpu"][i], a["drv_mem"][i], a["drv_gpu"][i]))
        for t in range(a["count"][i]):
            exp.append((i, t + 1, en[off[i] + t], a["exe_cpu"][i], a["exe_mem"][i], a["exe_gpu"][i]))
    exp = np.array(exp, np.int64)
    got = np.stack([rows[k].astype(np.int64) for k in ("app", "slot", "node", "cpu", "mem", "gpu")], axis=1)
    assert np.array_equal(got, exp)
    use_c = np.zeros(800, np.int64); use_m = np.zeros(800, np.int64)
    np.add.at(use_c, exp[:, 2], exp[:, 3]); np.add.at(use_m, exp[:, 2], exp[:, 4])
    fc, fm, fg = packer.get_snapshot()
    assert np.array_equal(fc, nodes["avail_cpu"] - use_c) and np.array_equal(fm, nodes["avail_mem"] - use_m)
    # the next batch packs against the charged snapshot without gp_set_snapshot
    nxt = synth.make_apps(200, seed=4)
    b = {k: nxt[k] for k in KEYS}
    from helpers import res_aos, assert_same_results
    for algo in (0, 1):
        got2 = packer.pack_batch(b, algo, 0)
        _, wd, we, woff, _ = oracle.closed_batch(algo, 0, fc, fm, fg, drv_order, exe_order, res_aos(b["drv_cpu"], b["drv_mem"], b["drv_gpu"]),
                                                 res_aos(b["exe_cpu"], b["exe_mem"], b["exe_gpu"]), b["count"], None, n_threads=4)
        assert_same_results(got2, (wd, we, woff), f"after reserve algo {algo}")
    # releasing every reservation restores the original availability, bit for bit
    packer.apply_usage_delta(exp[:, 2], exp[:, 3], exp[:, 4], exp[:, 5], sign=-1)
    rc, rm, rg = packer.get_snapshot()
    assert np.array_equal(rc, nodes["avail_cpu"]) and np.array_equal(rm, nodes["avail_mem"])
    got3 = packer.pack_batch(a, 0, 0)
    assert_same_results(got3, placed, "after release")


def test_reschedule_availability_double_counts_overhead(oracle, packer):
    """EXT/resource.go:638-643 bug for bug (SURVEY App. B7): nodes that carry a reservation lose their overhead twice in the
    availability the first-fit reschedule sees.  Device == the statement-by-statement restatement; and the node choice of
    a first-fit reschedule on that availability == the literal oracle's."""
    rng = np.random.default_rng(21)
    n, R = 500, 900
    names = node_names(n)
    alloc = [(rng.integers(8, 64, n) * 1000).astype(np.int64), (rng.integers(16, 256, n) << 30).astype(np.int64), rng.integers(0, 3, n).astype(np.int64)]
    over = [(rng.integers(0, 4, n) * 250).astype(np.int64), (rng.integers(0, 8, n) << 28).astype(np.int64), np.zeros(n, np.int64)]
    rnode = rng.integers(-1, n // 2, R).astype(np.int32)            # half of the nodes carry reservations; -1 = a node that left
    res = [(rng.integers(0, 5, R) * 500).astype(np.int64), (rng.integers(0, 9, R) << 29).astype(np.int64), (rng.integers(0, 4, R) == 0).astype(np.int64)]
    got = packer.build_reschedule_availability(alloc, over, rnode, res)
    want = oracle.reschedule_available(names, alloc, over, [names[i] if i >= 0 else "gone-%d" % t for t, i in enumerate(rnode)], res)
    for g_, w_ in zip(got, want):
        assert np.array_equal(g_, w_)
    plain, _ = packer.build_availability(alloc, over, rnode, res)
    has = np.zeros(n, bool); has[rnode[rnode >= 0]] = True
    assert np.array_equal(plain[0] - got[0], over[0] * has)         # exactly one extra overhead where a reservation exists


def _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, fifo, label):
    """Both single-AZ packers (and, for the FIFO loop, both accounting modes) on the device against the literal
    restatement with efficiencies -> [(algo, mode, zone, driver_node)] of the device runs."""
    n = len(cpu)
    names = node_names(n)
    labels = ["zone-%d" % z for z in zone_of]
    zones, eo, do, eoff, doff = _zone_groups(order_d, order_e, zone_of)
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"]); exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    runs = []
    for algo, oalgo in ((0, 2), (2, 5)):
        for mode in ((1, 2) if fifo else (0,)):
            cl = oracle.Cluster(names, cpu, mem, gpu, sched=(sc, sm, sg), zone=labels)
            packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
            packer.set_schedulable(sc, sm, sg)
            if fifo:
                _, wd, we, woff = cl.fifo(oalgo, mode, drv, exe, apps["count"], apps["young"], [names[i] for i in order_d],
                                          [names[i] for i in order_e], with_efficiencies=True)
                zone, gd, ge, goff, _ = packer.pack_fifo_zones(apps, algo, mode)
            else:
                wd, we, woff = cl.binpack_batch(oalgo, drv, exe, apps["count"], [names[i] for i in order_d], [names[i] for i in order_e],
                                                with_efficiencies=True, n_threads=4)
                zone, gd, ge, goff, _ = packer.pack_batch_zones(apps, algo)
            assert np.array_equal(goff, woff)
            bad = np.nonzero(gd != wd)[0]
            assert bad.size == 0, (label, algo, mode, bad[:5], gd[bad[:5]], wd[bad[:5]], zone[bad[:5]])
            for i in np.nonzero(wd >= 0)[0]:
                assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]]), (label, algo, mode, i)
                assert zone[i] == zones.index(zone_of[wd[i]]), (label, algo, mode, i)
            assert (zone[wd < 0] == -1).all()
            if fifo:
                fc, fm, fg = packer.get_snapshot()
                wc, wm, wg = cl.available()
                assert np.array_equal(fc, wc) and np.array_equal(fm, wm) and np.array_equal(fg, wg), (label, algo, mode)
            runs.append((algo, mode, zone, gd))
    return runs


def _many_zones(seed, Z, per, q):
    rng = np.random.default_rng(seed)
    n = Z * per
    cpu, mem, gpu = random_cluster(rng, n)
    sc = cpu + rng.integers(0, 9, n) * 250 + (rng.integers(0, 3, n) == 0) * 1
    sm = mem + rng.integers(0, 17, n) * (1 << 28)
    zone_of = rng.permutation(np.arange(n) % Z)               # every zone has nodes
    order_e = [int(i) for i in rng.permutation(n)]
    order_d = [int(i) for i in rng.permutation(n)]
    rank = {z: r for r, z in enumerate(_zone_groups(order_d, order_e, zone_of)[0])}
    late = np.array([rank[z] >= 32 for z in zone_of])         # more of these nodes in use: higher efficiencies, they win often
    sc, sm = sc + late * 16000, sm + late * (64 << 30)
    apps = random_apps(rng, q)
    apps["young"] = (rng.random(q) < 0.97).astype(np.uint8)
    return cpu, mem, gpu, sc, sm, gpu.clip(0), zone_of, order_d, order_e, apps


@pytest.mark.parametrize("Z", [16, 17, 33, 64])
def test_fifo_zones_beyond_one_warp(oracle, packer, Z):
    """gp_pack_fifo_zones strides the zones over 16 warps: winners packed by a warp other than 0 and by the second stride
    (z >= 16), up to the 64-zone limit of its shared-memory table."""
    cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps = _many_zones(5000 + Z, Z, 6, 120)
    runs = _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, True, f"Z={Z}")
    won = np.concatenate([zone[gd >= 0] for _, _, zone, gd in runs])
    assert (won % 16 != 0).any()                              # a warp other than 0
    if Z > 16:
        assert (won >= 16).any()                              # the second stride


@pytest.mark.parametrize("Z", [31, 32, 33, 70])
def test_batch_zones_across_warp_steps(oracle, packer, Z):
    """gp_zone_choose walks the zones 32 per warp step and applies the tie rule across steps."""
    cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps = _many_zones(5100 + Z, Z, 5, 150)
    runs = _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, sc, sm, sg, zone_of, order_d, order_e, apps, False, f"Z={Z}")
    won = np.concatenate([zone[gd >= 0] for _, _, zone, gd in runs])
    assert (won >= 32).any() if Z > 32 else (won >= 24).any()


@pytest.mark.parametrize("first_fit_zone", [0, 31])
def test_zone_ties_go_to_the_first_zone(oracle, packer, first_fit_zone):
    """40 zones, identical from `first_fit_zone` on (the zones before it cannot host a driver): every tie of the averages
    goes to the first zone (strict '<', single_az.go:91-94).  With 31, the tie spans the 32-zone step of gp_zone_choose
    and the two warp strides of gp_pack_fifo_zones."""
    Z, per = 40, 3
    n = Z * per
    zone_of = np.repeat(np.arange(Z), per)
    cpu = np.where(zone_of < first_fit_zone, 200, np.tile([8000, 6000, 4000], Z)).astype(np.int64)
    mem = np.tile([32 << 30, 24 << 30, 16 << 30], Z).astype(np.int64)
    gpu = np.zeros(n, np.int64)
    sc, sm = cpu + 8000, mem + (32 << 30)
    order = list(range(n))
    q = 24
    i = np.arange(q)
    apps = {"drv_cpu": np.full(q, 1000, np.int64), "drv_mem": np.full(q, 1 << 30, np.int64), "drv_gpu": np.zeros(q, np.int64),
            "exe_cpu": 500 * (1 + i % 3), "exe_mem": (1 << 30) * (1 + i % 2), "exe_gpu": np.zeros(q, np.int64),
            "count": (1 + i % 4).astype(np.int32), "young": np.ones(q, np.uint8)}
    runs = _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, sc, sm, gpu, zone_of, order, order, apps, False, "ties batch")
    for _, _, zone, gd in runs:
        assert (gd >= 0).all() and (zone == first_fit_zone).all()
    runs = _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, sc, sm, gpu, zone_of, order, order, apps, True, "ties fifo")
    for _, _, zone, gd in runs:
        assert zone[0] == first_fit_zone


@pytest.mark.parametrize("young", [0, 1])
def test_zero_efficiency_picks_no_zone(oracle, packer, young):
    """A driver-only application with zero requests on untouched nodes packs with an average efficiency of exactly 0.0:
    chooseBestResult keeps nothing (best starts at 0.0, strict '<'), so it fits nowhere; in the FIFO loop a non-young one
    then blocks the queue."""
    n = 12
    cpu = np.full(n, 8000, np.int64); mem = np.full(n, 32 << 30, np.int64); gpu = np.zeros(n, np.int64)
    zone_of = np.arange(n) % 3
    order = list(range(n))
    apps = {"drv_cpu": np.array([0, 1000, 1000], np.int64), "drv_mem": np.array([0, 1 << 30, 1 << 30], np.int64),
            "drv_gpu": np.zeros(3, np.int64), "exe_cpu": np.array([1000, 2000, 1000], np.int64),
            "exe_mem": np.full(3, 2 << 30, np.int64), "exe_gpu": np.zeros(3, np.int64),
            "count": np.array([0, 2, 1], np.int32), "young": np.array([young, 0, 0], np.uint8)}
    runs = _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, cpu, mem, gpu, zone_of, order, order, apps, True, "zero eff fifo")
    for _, _, zone, gd in runs:
        assert gd[0] == -1 and zone[0] == -1
        assert (gd[1:] >= 0).all() if young else (gd[1:] == -2).all()
    runs = _zone_literal_vs_device(oracle, packer, cpu, mem, gpu, cpu, mem, gpu, zone_of, order, order, apps, False, "zero eff batch")
    for _, _, zone, gd in runs:
        assert gd[0] == -1 and (gd[1:] >= 0).all()


def test_fifo_zones_refuses_more_than_64(packer, gangpack):
    n = 65 * 2
    cpu = np.full(n, 8000, np.int64); mem = np.full(n, 32 << 30, np.int64); gpu = np.zeros(n, np.int64)
    order = list(range(n))
    _, eo, do, eoff, doff = _zone_groups(order, order, np.arange(n) % 65)
    packer.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    packer.set_schedulable(cpu, mem, gpu)
    apps = random_apps(np.random.default_rng(1), 4)
    with pytest.raises(gangpack.native.GangpackError) as e:
        packer.pack_fifo_zones(apps, 0, 1)
    assert e.value.status == 1
    zone, gd, _, _, _ = packer.pack_batch_zones(apps, 0)          # the independent form has no zone limit
    assert (gd >= 0).any() and (zone[gd >= 0] < 65).all()
