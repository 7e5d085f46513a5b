"""gp_packing_efficiency: computeAvgPackingEfficiencyForResult over every node of the snapshot, exactly summed, on the device.

Checked against
- the restatement: math.fsum over pyref.compute_packing_efficiency of EVERY node (reserved per the algo rule), bit for bit;
- the literal oracle's orc_binpack(with_efficiencies = 1), which sums in insertion order: within the recursive-summation
  bound gamma_{N-1} * sum|t_i| / len + 2 ulp, and bit for bit on clusters where every partial sum is exact;
for every packer (tightly-pack, distribute-evenly, minimal-fragmentation, the single-AZ winners, the az-aware winners and
fallback rows), the two FIFO recipes, the reservation recipe, order invariance, a 100 000-row batch, state and refusals."""
import math

import numpy as np
import pytest

from helpers import random_apps, res_aos

pytestmark = pytest.mark.gpu

G = 1 << 30
INDEPENDENT, FIFO_REFERENCE, FIFO_EXACT = 0, 1, 2
TIGHTLY, EVENLY, MINFRAG = 0, 1, 2
ORC_ALGO = {TIGHTLY: 0, EVENLY: 1, MINFRAG: 4}


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


# ---- clusters ---------------------------------------------------------------------------------------------------------
def make_cluster(rng, n, pow2=False):
    """(avail[3], sched[3]) with overcommitted nodes, zero / negative schedulable values, mixed GPU and non-GPU nodes and CPU
    that is not a multiple of 1000.  pow2: schedulable values are powers of two and usage is coarse, so every partial sum
    of every term is exact in float64."""
    if pow2:
        sc = 1000 * (1 << rng.integers(2, 7, n))
        sm = (1 << rng.integers(30, 39, n)).astype(np.int64)
        sg = np.where(rng.random(n) < 0.4, 1 << rng.integers(0, 4, n), 0)
        ac = sc - 1000 * rng.integers(-4, 2 * (sc // 1000) + 1)
        am = sm - (1 << 20) * rng.integers(-64, 2 * (sm >> 20) + 1)
        ag = sg - rng.integers(-1, 2 * sg + 1)
    else:
        sc = rng.integers(1, 64, n) * 1000 + np.where(rng.random(n) < 0.5, rng.integers(0, 1000, n), 0)
        sc = np.where(rng.random(n) < 0.05, 0, np.where(rng.random(n) < 0.05, -rng.integers(1, 3000, n), sc))
        sm = rng.integers(1, 256, n) * G + rng.integers(0, 1 << 20, n)
        sm = np.where(rng.random(n) < 0.05, 0, np.where(rng.random(n) < 0.05, -rng.integers(1, G, n), sm))
        sg = np.where(rng.random(n) < 0.3, rng.integers(1, 9, n), 0)
        sg = np.where(rng.random(n) < 0.03, -1, sg)
        ac = sc - rng.integers(-2000, np.maximum(sc, 0) + 5000)          # some above sched, some overcommitted
        am = sm - rng.integers(-G, np.maximum(sm, 0) + 4 * G)
        ag = sg - rng.integers(-1, np.maximum(sg, 0) + 3)
    f = lambda x: np.asarray(x, np.int64)
    return [f(ac), f(am), f(ag)], [f(sc), f(sm), f(sg)]


def fit_apps(rng, q, gpus=True):
    a = random_apps(rng, q, gpus=gpus, big_counts=True)
    return a


# ---- the restatement ----------------------------------------------------------------------------------------------------
class Restated:
    """the reference's per-node terms of every node for one availability; rows swap in the reserved terms and fsum"""

    def __init__(self, avail, sched):
        from oracle import pyref
        self.pyref = pyref
        self.avail = [[int(x) for x in col] for col in avail]
        self.sched = [[int(x) for x in col] for col in sched]
        self.n = len(self.avail[0])
        self.base = [self.terms(i, None) for i in range(self.n)]

    def terms(self, i, reserved, back=(0, 0, 0)):
        av = tuple(self.avail[r][i] + back[r] for r in range(3))
        sc = tuple(self.sched[r][i] for r in range(3))
        c, m, g = self.pyref.compute_packing_efficiency(av, sc, reserved)
        return c, m, g, max(g, max(c, m))

    def avg(self, reserved, back=None):
        t = list(self.base)
        for i in set(reserved) | set(back or {}):
            t[i] = self.terms(i, reserved.get(i), (back or {}).get(i, (0, 0, 0)))
        L = max(float(self.n), 1.0)
        gpu = [t[i][2] for i in range(self.n) if self.sched[2][i] != 0]
        return (math.fsum(x[0] for x in t) / L, math.fsum(x[1] for x in t) / L,
                1.0 if not gpu else math.fsum(gpu) / float(len(gpu)), math.fsum(x[3] for x in t) / L), t


def reserved_of(algo, drv, exe, d, nodes):
    if algo == MINFRAG:
        return {d: drv}
    r = {d: drv}
    for n in nodes:
        o = r.get(n, (0, 0, 0))
        r[n] = (o[0] + exe[0], o[1] + exe[1], o[2] + exe[2])
    return r


def app_res(apps, i):
    return ((int(apps["drv_cpu"][i]), int(apps["drv_mem"][i]), int(apps["drv_gpu"][i])),
            (int(apps["exe_cpu"][i]), int(apps["exe_mem"][i]), int(apps["exe_gpu"][i])))


def within_bound(dev, orc, t):
    """|dev - orc| <= gamma_{m-1} * sum|t| / len + 2 ulp(orc) per component (m = number of summed terms)"""
    u = 2.0 ** -53
    cols = [[x[0] for x in t], [x[1] for x in t], [x[2] for x in t if x[4] != 0], [x[3] for x in t]]
    for j, col in enumerate(cols):
        m = len(col)
        if j == 2 and m == 0:
            assert dev[j] == orc[j] == 1.0
            continue
        L = float(m) if j == 2 else max(float(len(t)), 1.0)
        gam = (m - 1) * u / (1 - (m - 1) * u) if m > 1 else 0.0
        bound = gam * math.fsum(abs(x) for x in col) / L + 2 * math.ulp(orc[j])
        assert abs(dev[j] - orc[j]) <= bound, (j, dev[j], orc[j], bound)


def bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def check_rows(dev, apps, placed, algo_of_row, rs, rows, label):
    drv, exe, off = placed
    for i in rows:
        if drv[i] < 0:
            assert (dev[i] == 0.0).all(), (label, i)
            continue
        dr, er = app_res(apps, i)
        want, _ = rs.avg(reserved_of(algo_of_row(i), dr, er, int(drv[i]), [int(x) for x in exe[off[i]:off[i + 1]]]))
        assert np.array_equal(bits(dev[i]), bits(want)), (label, i, dev[i], want)


def names_of(n):
    return ["node-%06d" % i for i in range(n)]


# ---- every packer through gp_pack_batch -------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [10, 1000, 10000])
@pytest.mark.parametrize("algo", [TIGHTLY, EVENLY, MINFRAG])
def test_pack_batch_packers(packer, oracle, n, algo):
    rng = np.random.default_rng(n * 7 + algo)
    avail, sched = make_cluster(rng, n)
    order = rng.permutation(n).astype(np.int32)
    dorder = order[rng.random(n) < 0.8]
    packer.set_snapshot(*avail, order, dorder)
    packer.set_schedulable(*sched)
    q = 300
    apps = fit_apps(rng, q)
    placed = packer.pack_batch(apps, algo)
    dev = packer.packing_efficiency(apps, placed, algo)
    assert dev.shape == (q, 4)
    rs = Restated(avail, sched)
    rows = list(range(q)) if n <= 1000 else list(rng.choice(q, 40, replace=False))
    check_rows(dev, apps, placed, lambda i: algo, rs, rows, f"pack_batch algo={algo} n={n}")
    # the literal oracle (insertion-order sums) on a sample: same placement, averages within the summation bound
    names = names_of(n)
    cl = oracle.Cluster(names, *avail, sched=sched)
    for i in rows[:25]:
        dr, er = app_res(apps, i)
        ok, dn, en, eff = cl.binpack(ORC_ALGO[algo], dr, er, int(apps["count"][i]), [names[j] for j in dorder],
                                     [names[j] for j in order], with_efficiencies=True)
        drv, exe, off = placed
        assert ok == (drv[i] >= 0), (algo, i)
        if not ok:
            continue
        assert dn == names[drv[i]] and en == [names[j] for j in exe[off[i]:off[i + 1]]]
        _, t = rs.avg(reserved_of(algo, dr, er, int(drv[i]), [int(x) for x in exe[off[i]:off[i + 1]]]))
        within_bound(dev[i], eff, [x + (sched[2][k],) for k, x in enumerate(t)])


@pytest.mark.parametrize("algo", [TIGHTLY, EVENLY, MINFRAG])
def test_exactly_representable_equals_oracle_bitwise(packer, oracle, algo):
    rng = np.random.default_rng(40 + algo)
    n = 2000
    avail, sched = make_cluster(rng, n, pow2=True)
    order = rng.permutation(n).astype(np.int32)
    packer.set_snapshot(*avail, order, order)
    packer.set_schedulable(*sched)
    apps = fit_apps(rng, 60)
    for k in ("drv_cpu", "exe_cpu"):
        apps[k] = (apps[k] // 1000) * 1000                                 # whole cores: CPU terms stay dyadic
    apps["drv_mem"] = (apps["drv_mem"] >> 20) << 20
    apps["exe_mem"] = (apps["exe_mem"] >> 20) << 20
    placed = packer.pack_batch(apps, algo)
    dev = packer.packing_efficiency(apps, placed, algo)
    names = names_of(n)
    cl = oracle.Cluster(names, *avail, sched=sched)
    onames = [names[j] for j in order]
    placed_rows = 0
    for i in range(len(apps["count"])):
        dr, er = app_res(apps, i)
        ok, dn, en, eff = cl.binpack(ORC_ALGO[algo], dr, er, int(apps["count"][i]), onames, onames, with_efficiencies=True)
        if ok:
            placed_rows += 1
            assert np.array_equal(bits(dev[i]), bits(eff)), (algo, i, dev[i], eff)
    assert placed_rows > 10


# ---- the zone packers ---------------------------------------------------------------------------------------------------
def zone_snapshot(packer, rng, n, Z, avail, sched):
    """Z zones, every zone with driver and executor candidates, groups in first-appearance order of the driver order."""
    zone = rng.integers(0, Z, n)
    zone[:Z] = np.arange(Z)
    dorder = rng.permutation(n).astype(np.int32)
    eorder = rng.permutation(n).astype(np.int32)
    zones_in_order = list(dict.fromkeys(int(zone[v]) for v in dorder))
    eo, do, eoff, doff = [], [], [0], [0]
    for z in zones_in_order:
        eo += [int(v) for v in eorder if zone[v] == z]
        do += [int(v) for v in dorder if zone[v] == z]
        eoff.append(len(eo)); doff.append(len(do))
    packer.set_snapshot(*avail, np.array(eo, np.int32), np.array(do, np.int32), np.array(eoff, np.int32), np.array(doff, np.int32))
    packer.set_schedulable(*sched)
    return dorder, eorder, len(zones_in_order)


@pytest.mark.parametrize("n", [10, 1000])
def test_single_az_and_az_aware_winners_and_fallback(packer, n):
    rng = np.random.default_rng(70 + n)
    avail, sched = make_cluster(rng, n)
    avail[0] = np.abs(avail[0]) + 8000                                    # room enough that zones win
    avail[1] = np.abs(avail[1]) + 16 * G
    Z = 3
    dorder, eorder, nz = zone_snapshot(packer, rng, n, Z, avail, sched)
    rs = Restated(avail, sched)
    q = 200
    apps = fit_apps(rng, q)
    apps["count"] = np.where(rng.random(q) < 0.3, rng.integers(n // 3 + 1, n + 2, q), apps["count"]).astype(np.int32)
    for algo in (TIGHTLY, MINFRAG):
        zone, drv, exe, off, _ = packer.pack_batch_zones(apps, algo)
        placed = (drv, exe, off)
        dev = packer.packing_efficiency(apps, placed, algo)
        check_rows(dev, apps, placed, lambda i: algo, rs, range(q), f"single-az algo={algo} n={n}")
    zone, drv, exe, off, _ = packer.pack_batch_az_aware(apps, eorder, dorder, nz)
    fallback = (zone == -1) & (drv >= 0)
    winners = zone >= 0
    assert winners.any()
    if n == 1000:
        assert fallback.any()
    placed = (drv, exe, off)
    dev = packer.packing_efficiency(apps, placed, TIGHTLY)
    check_rows(dev, apps, placed, lambda i: TIGHTLY, rs, range(q), f"az-aware n={n}")


# ---- order invariance ---------------------------------------------------------------------------------------------------
def test_node_table_permutation_is_bit_identical(packer):
    rng = np.random.default_rng(90)
    n = 5000
    avail, sched = make_cluster(rng, n)
    order = rng.permutation(n).astype(np.int32)
    packer.set_snapshot(*avail, order, order)
    packer.set_schedulable(*sched)
    apps = fit_apps(rng, 400)
    placed = packer.pack_batch(apps, TIGHTLY)
    a = packer.packing_efficiency(apps, placed, TIGHTLY)
    perm = rng.permutation(n)                                             # new index of old node v = inv[v]
    inv = np.empty(n, np.int64); inv[perm] = np.arange(n)
    packer.set_snapshot(*[c[perm] for c in avail], inv[order].astype(np.int32), inv[order].astype(np.int32))
    packer.set_schedulable(*[c[perm] for c in sched])
    drv, exe, off = placed
    remapped = (np.where(drv >= 0, inv[np.maximum(drv, 0)], drv).astype(np.int32), inv[exe].astype(np.int32), off)
    b = packer.packing_efficiency(apps, remapped, TIGHTLY)
    assert np.array_equal(bits(a), bits(b))
    assert packer.pack_batch(apps, TIGHTLY)[0].tolist() == remapped[0].tolist()


# ---- the FIFO recipes ---------------------------------------------------------------------------------------------------
def usage_case(rng, n):
    alloc = [rng.integers(2, 65, n) * 1000 + rng.integers(0, 2, n) * 500, rng.integers(4, 257, n) * G,
             (rng.random(n) < 0.3) * rng.integers(1, 9, n)]
    over = [rng.integers(0, 3, n) * 300, rng.integers(0, 3, n) * (1 << 28), np.zeros(n, np.int64)]
    over[0] = np.where(rng.random(n) < 0.03, alloc[0] + 500, over[0])     # overhead above allocatable: negative sched
    R = 3 * n
    rnode = rng.integers(-1, n, R).astype(np.int32)
    res = [rng.integers(0, 9, R) * 500, rng.integers(0, 9, R) * (1 << 29), (rng.random(R) < 0.1).astype(np.int64)]
    return [np.asarray(x, np.int64) for x in alloc], [np.asarray(x, np.int64) for x in over], rnode, [np.asarray(x, np.int64) for x in res]


def one_app(apps, i):
    return {k: np.asarray(v)[i:i + 1] for k, v in apps.items() if k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "young")}


@pytest.mark.parametrize("mode", [FIFO_REFERENCE, FIFO_EXACT])
@pytest.mark.parametrize("algo", [TIGHTLY, EVENLY])
def test_fifo_recipe_prepare_cluster(gangpack, packer, oracle, mode, algo):
    rng = np.random.default_rng(100 + 10 * mode + algo)
    n, q = 1000, 120
    alloc, over, rnode, res = usage_case(rng, n)
    aux = gangpack.GangPacker()
    try:
        av, sc = aux.build_availability(alloc, over, rnode, res)
        d_order, e_order = aux.potential_nodes(av[0], av[1], avail_gpu=av[2])
    finally:
        aux.close()
    apps = fit_apps(rng, q)
    apps["young"] = np.ones(q, np.uint8)
    # the queue ends with a driver that fits: cut it after the last placed entry (FIFO decisions do not look ahead)
    packer.prepare_cluster(alloc, over, rnode, res)
    last = int(np.nonzero(packer.pack_batch(apps, algo, mode)[0] >= 0)[0][-1])
    apps = {k: v[:last + 1] for k, v in apps.items()}
    packer.prepare_cluster(alloc, over, rnode, res)
    drv, exe, off = packer.pack_batch(apps, algo, mode)
    assert drv[last] >= 0
    dev = packer.packing_efficiency(one_app(apps, last), (drv[last:], exe[off[last]:off[last + 1]], np.array([0, off[last + 1] - off[last]])),
                                    algo, charged=mode)
    # the availability orc_fifo leaves after the first q - 1 entries
    names = names_of(n)
    cl = oracle.Cluster(names, *av, sched=sc)
    sub = {k: v[:last] for k, v in apps.items()}
    oracle_res = lambda a: (res_aos(a["drv_cpu"], a["drv_mem"], a["drv_gpu"]), res_aos(a["exe_cpu"], a["exe_mem"], a["exe_gpu"]))
    od, oe = oracle_res(sub)
    _, odn, _, _ = cl.fifo(algo, mode, od, oe, sub["count"], sub["young"], [names[j] for j in d_order], [names[j] for j in e_order])
    assert np.array_equal(odn, drv[:last])
    rs = Restated(cl.available(), sc)
    dr, er = app_res(apps, last)
    nodes = [int(x) for x in exe[off[last]:off[last + 1]]]
    want, _ = rs.avg(reserved_of(algo, dr, er, int(drv[last]), nodes))
    assert np.array_equal(bits(dev[0]), bits(want)), (dev[0], want)
    # the same call without the add-back would see the driver twice: it differs whenever the placement moved anything
    charged = packer.packing_efficiency(one_app(apps, last), (drv[last:], exe[off[last]:off[last + 1]], np.array([0, len(nodes)])), algo)
    want_charged, _ = Restated(packer.get_snapshot(), sc).avg(reserved_of(algo, dr, er, int(drv[last]), nodes))
    assert np.array_equal(bits(charged[0]), bits(want_charged))


@pytest.mark.parametrize("mode", [FIFO_REFERENCE, FIFO_EXACT])
def test_fifo_recipe_az_aware(gangpack, packer, oracle, mode):
    rng = np.random.default_rng(200 + mode)
    n, q, Z = 1000, 80, 3
    alloc, over, rnode, res = usage_case(rng, n)
    zid = rng.integers(0, Z, n).astype(np.int32)
    seen = {}
    zid = np.array([seen.setdefault(int(z), len(seen)) for z in zid], np.int32)
    aux = gangpack.GangPacker()
    try:
        av, sc = aux.build_availability(alloc, over, rnode, res)
        d_order, e_order = aux.potential_nodes(av[0], av[1], zone_id=zid, n_zones=len(seen), avail_gpu=av[2])
    finally:
        aux.close()
    apps = fit_apps(rng, q)
    apps["young"] = np.ones(q, np.uint8)
    packer.prepare_cluster_zones(alloc, over, rnode, res, zone_id=zid, n_zones=len(seen))
    last = int(np.nonzero(packer.pack_fifo_az_aware(apps, mode)[1] >= 0)[0][-1])
    apps = {k: v[:last + 1] for k, v in apps.items()}
    packer.prepare_cluster_zones(alloc, over, rnode, res, zone_id=zid, n_zones=len(seen))
    zone, drv, exe, off, _ = packer.pack_fifo_az_aware(apps, mode)
    assert drv[last] >= 0
    nodes = [int(x) for x in exe[off[last]:off[last + 1]]]
    dev = packer.packing_efficiency(one_app(apps, last), (drv[last:], exe[off[last]:off[last + 1]], np.array([0, len(nodes)])),
                                    TIGHTLY, charged=mode)
    names = names_of(n)
    cl = oracle.Cluster(names, *av, sched=sc, zone=["zone-%d" % z for z in zid])
    sub = {k: v[:last] for k, v in apps.items()}
    od = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"])
    oe = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
    _, odn, _, _ = cl.fifo(3, mode, od, oe, sub["count"], sub["young"], [names[j] for j in d_order], [names[j] for j in e_order])
    assert np.array_equal(odn, drv[:last])
    dr, er = app_res(apps, last)
    want, _ = Restated(cl.available(), sc).avg(reserved_of(TIGHTLY, dr, er, int(drv[last]), nodes))
    assert np.array_equal(bits(dev[0]), bits(want)), (dev[0], want)


@pytest.mark.parametrize("algo", [TIGHTLY, EVENLY, MINFRAG])
def test_reserve_recipe(packer, algo):
    rng = np.random.default_rng(300 + algo)
    n = 3000
    avail, sched = make_cluster(rng, n)
    order = rng.permutation(n).astype(np.int32)
    packer.set_snapshot(*avail, order, order)
    packer.set_schedulable(*sched)
    apps = fit_apps(rng, 40)
    checked = 0
    for i in range(40):
        a = one_app(apps, i)
        placed = packer.pack_batch(a, algo)
        if placed[0][0] < 0:
            continue
        before = packer.packing_efficiency(a, placed, algo)
        packer.reserve_placements(a, placed, subtract=True)
        after = packer.packing_efficiency(a, placed, algo, charged=FIFO_EXACT)
        assert np.array_equal(bits(before), bits(after)), (algo, i)
        checked += 1
    assert checked > 5


# ---- batch, state, refusals ----------------------------------------------------------------------------------------------
def test_batch_of_100k_rows_equals_single_calls(packer):
    rng = np.random.default_rng(400)
    n, q = 1000, 100_000
    avail, sched = make_cluster(rng, n)
    order = rng.permutation(n).astype(np.int32)
    packer.set_snapshot(*avail, order, order)
    packer.set_schedulable(*sched)
    apps = fit_apps(rng, q)
    drv, exe, off = packer.pack_batch(apps, EVENLY)
    drv = drv.copy()
    drv[rng.random(q) < 0.05] = -1                                        # rows without a placement
    batch = packer.packing_efficiency(apps, (drv, exe, off), EVENLY)
    for i in range(q):
        one = packer.packing_efficiency(one_app(apps, i), (drv[i:i + 1], exe[off[i]:off[i + 1]], np.array([0, off[i + 1] - off[i]])), EVENLY)
        assert np.array_equal(bits(one[0]), bits(batch[i])), i
    assert (batch[drv < 0] == 0.0).all()
    rs = Restated(avail, sched)
    check_rows(batch, apps, (drv, exe, off), lambda i: EVENLY, rs, list(rng.choice(q, 30, replace=False)), "100k sample")


def test_state_is_untouched(packer):
    rng = np.random.default_rng(500)
    n = 2000
    avail, sched = make_cluster(rng, n)
    order = rng.permutation(n).astype(np.int32)
    packer.set_snapshot(*avail, order, order[: n // 2])
    packer.set_schedulable(*sched)
    apps = fit_apps(rng, 500)
    placed = packer.pack_batch(apps, TIGHTLY, FIFO_EXACT)
    snap0, stats0 = packer.get_snapshot(), packer.stats()
    drv = placed[0].copy()
    drv[::7] = -1
    out = packer.packing_efficiency(apps, (drv, placed[1], placed[2]), TIGHTLY)
    assert (out[::7] == 0.0).all() and np.signbit(out[::7]).sum() == 0
    snap1, stats1 = packer.get_snapshot(), packer.stats()
    for x, y in zip(snap0, snap1):
        assert np.array_equal(x, y)
    assert stats0 == stats1


def test_refusals(gangpack, packer):
    rng = np.random.default_rng(600)
    apps = fit_apps(rng, 2)
    apps["count"] = np.array([2, 1], np.int32)
    placed = (np.array([0, 1], np.int32), np.array([0, 1, 2], np.int32), np.array([0, 2, 3], np.int64))
    fresh = gangpack.GangPacker()
    try:
        with pytest.raises(gangpack.GangpackError) as e:
            fresh.packing_efficiency(apps, placed, TIGHTLY)
        assert e.value.status == 4
        n = 8
        avail, sched = make_cluster(rng, n)
        order = np.arange(n, dtype=np.int32)
        fresh.set_snapshot(*avail, order, order)
        with pytest.raises(gangpack.GangpackError) as e:                 # no SchedulableResources
            fresh.packing_efficiency(apps, placed, TIGHTLY)
        assert e.value.status == 1 and "SchedulableResources" in str(e.value)
        fresh.set_schedulable(*sched)
        fresh.packing_efficiency(apps, placed, TIGHTLY)
        bad = (placed[0], np.array([0, 9, 2], np.int32), placed[2])
        with pytest.raises(gangpack.GangpackError) as e:
            fresh.packing_efficiency(apps, bad, TIGHTLY)
        assert e.value.status == 1 and "out of range" in str(e.value)
        with pytest.raises(gangpack.GangpackError) as e:
            fresh.packing_efficiency(apps, (np.array([8, 1], np.int32), placed[1], placed[2]), TIGHTLY)
        assert e.value.status == 1
        with pytest.raises(gangpack.GangpackError) as e:
            fresh.packing_efficiency(apps, placed, TIGHTLY, charged=FIFO_EXACT)
        assert e.value.status == 1 and "n_apps" in str(e.value)
        with pytest.raises(gangpack.GangpackError) as e:                 # cap too small
            fresh.packing_efficiency(apps, (placed[0], placed[1][:2], placed[2]), TIGHTLY)
        assert e.value.status == 5
        big = dict(apps)
        big["exe_mem"] = np.array([1 << 60, 1], np.int64)                 # two executors on node 0: 2^61 reserved there
        big_placed = (placed[0], np.array([0, 0, 2], np.int32), placed[2])
        with pytest.raises(gangpack.GangpackError) as e:
            fresh.packing_efficiency(big, big_placed, TIGHTLY)
        assert e.value.status == 6
        fresh.packing_efficiency(big, big_placed, MINFRAG)                # minimal-fragmentation reserves the driver only
        # the zone entry points keep refusing a gp_prepare_cluster snapshot
        alloc, over, rnode, res = usage_case(rng, 16)
        fresh.prepare_cluster(alloc, over, rnode, res)
        fresh.packing_efficiency(apps, (np.array([0, 1], np.int32), placed[1], placed[2]), TIGHTLY)
        with pytest.raises(gangpack.GangpackError) as e:
            fresh.pack_batch_zones(apps, TIGHTLY)
        assert e.value.status == 1 and "gp_set_schedulable first" in str(e.value)
    finally:
        fresh.close()
