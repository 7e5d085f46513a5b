"""gp_prepare_cluster_groups: reservations -> availability -> PotentialNodes per instance group -> the plain multi-group
snapshot of tightly-pack / distribute-evenly / minimal-fragmentation, on the device; and gp_packing_efficiency_groups, the
Predicate's metric averaged over each application's instance group.  Checked:
- identity: each instance group's orders, offsets, counts and undefined ties equal gp_prepare_cluster + gp_potential_nodes
  on a second context holding only that instance group's sub-table, mapped back; instance_group = NULL is gp_prepare_cluster;
- FIFO bit for bit (both packers, both modes, skip flags) against the host recipe and, per instance group, against the
  literal oracle loop; independent batches against the per-sub-table results;
- the state rules and refusals;
- the per-instance-group efficiency against gp_packing_efficiency on the sub-table's context."""
import numpy as np
import pytest

import frontend_ref as fr
from helpers import random_apps
from oracle import pyref
from test_gpu_prepare_zones import G as GIB, sort_args
from test_gpu_prepare_zones_groups import alone, groups_case, packer, prepare_groups, sub_table  # noqa: F401 (fixtures)
from test_zone_layout_model import AZ_AWARE

pytestmark = pytest.mark.gpu

ALGO_NAME = {0: "tightly-pack", 1: "distribute-evenly", 2: "minimal-fragmentation"}
MODE_NAME = {1: "reference", 2: "exact"}
_CASE = object()


def prep(p, c, ig=_CASE, G=None, orders=True):
    return p.prepare_cluster_groups(c["alloc"], c["over"], c["rnode"], c["res"], c["ig"] if ig is _CASE else ig,
                                    c["G"] if G is None else G, *sort_args(c), orders=orders)


def sub_orders(p, c, idx, av):
    """PotentialNodes of one instance group on its sub-table (device, second context) -> (drv, exe, ties) as sub indices"""
    s = sub_table(c, idx)
    d, e = p.potential_nodes(av[0][idx], av[1][idx], *sort_args(s), avail_gpu=av[2][idx])
    return d, e, p.undefined_ties, s


def check_identity(packer, alone, c, label):
    got = prep(packer, c)
    G = c["G"]
    av, _ = alone.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    assert got["exec_off"][0] == 0 and got["drv_off"][0] == 0, label
    tot = 0
    for i in range(G):
        idx = np.nonzero(c["ig"] == i)[0]
        e0, e1, d0, d1 = (int(x) for x in (got["exec_off"][i], got["exec_off"][i + 1], got["drv_off"][i], got["drv_off"][i + 1]))
        if idx.size == 0:
            assert e0 == e1 and d0 == d1 and got["ig_undefined_ties"][i] == 0, (label, i)
            continue
        d, e, ties, s = sub_orders(alone, c, idx, av)
        nd, ne = alone.prepare_cluster(s["alloc"], s["over"], s["rnode"], s["res"], *sort_args(s))
        assert (nd, ne) == (len(d), len(e)) == (d1 - d0, e1 - e0), (label, i)
        assert list(got["drv_order"][d0:d1]) == list(idx[d]) and list(got["exec_order"][e0:e1]) == list(idx[e]), (label, i)
        assert got["ig_undefined_ties"][i] == ties, (label, i)
        tot += ties
    assert got["undefined_ties"] == tot, label
    assert (got["n_driver"], got["n_executor"]) == (got["drv_off"][G], got["exec_off"][G]), label
    for x, y in zip(packer.get_snapshot(), av):
        assert np.array_equal(x, y), label
    return got


@pytest.mark.parametrize("G,n,Z", [(1, 400, 5), (2, 600, 4), (7, 1500, 9), (140, 4000, 6)])
def test_identity(packer, alone, G, n, Z):
    c = groups_case(1700 + G, n, G, Z, empty=(G - 1,) if G > 2 else ())
    check_identity(packer, alone, c, G)


def test_identity_ties_shared_zones_and_sort_tile(packer, alone):
    """instance group 0: equal nodes spread evenly over shared zone ids (every zone total ties, GPU ties undefined);
    instance groups 1 and 2 hold more than 4 096 nodes each (their orders cross the sort tile); label re-sorts throughout"""
    c = groups_case(1720, 9500, 3, 4, none_p=0.02)
    ig = c["ig"]
    ig[:300] = 0
    ig[300:] = np.where(ig[300:] == 0, 1 + np.arange(len(ig) - 300) % 2, ig[300:])
    zero = np.nonzero(ig == 0)[0]
    c["zid"][zero] = np.arange(len(zero)) % 4
    c["alloc"][0][zero] = 8000; c["alloc"][1][zero] = 32 * GIB; c["alloc"][2][zero] = np.arange(len(zero)) % 3
    c["over"][0][zero] = 0; c["over"][1][zero] = 0
    c["rnode"][np.isin(c["rnode"], zero)] = -1
    assert min((ig == 1).sum(), (ig == 2).sum()) > 4096
    got = check_identity(packer, alone, c, "ties")
    assert got["ig_undefined_ties"][0] > 0


def test_null_instance_group_is_prepare_cluster(packer, alone):
    c = groups_case(1730, 1200, 1, 6)
    rng = np.random.default_rng(1731)
    apps = random_apps(rng, 300, gpus=True)
    for G in (1, 3):
        got = prep(packer, c, ig=None, G=G)
        nd, ne = alone.prepare_cluster(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c))
        av, _ = alone.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
        d, e = alone.potential_nodes(av[0], av[1], *sort_args(c), avail_gpu=av[2])
        assert (got["n_driver"], got["n_executor"]) == (nd, ne)
        assert list(got["drv_order"]) == list(d) and list(got["exec_order"]) == list(e)
        assert list(got["exec_off"]) == [0] + [ne] * G and list(got["drv_off"]) == [0] + [nd] * G
        assert got["undefined_ties"] == alone.undefined_ties == got["ig_undefined_ties"][0]
        for algo in (0, 1, 2):
            for mode in ((0, 1, 2) if algo < 2 else (0,)):
                prep(packer, c, ig=None, G=G, orders=False)
                alone.prepare_cluster(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c))
                a, b = packer.pack_batch(apps, algo, mode), alone.pack_batch(apps, algo, mode)
                same_results(a, b, (G, algo, mode))
                for x, y in zip(packer.get_snapshot(), alone.get_snapshot()):
                    assert np.array_equal(x, y)


# ---- packing from the prepared snapshot ---------------------------------------------------------------------------------
def same_results(a, b, label):
    (da, ea, oa), (db, eb, ob) = a, b
    assert np.array_equal(oa, ob) and np.array_equal(da, db), (label, np.nonzero(da != db)[0][:5])
    for j in np.nonzero(da >= 0)[0]:
        assert np.array_equal(ea[oa[j]:oa[j + 1]], eb[ob[j]:ob[j + 1]]), (label, j)


def host_recipe(p, c):
    """gp_build_availability, gp_potential_nodes per sub-table, the orders concatenated, gp_set_snapshot -> (av, sc, orders)"""
    av, sc = p.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    eo, do, eoff, doff, orders = [], [], [0], [0], []
    for i in range(c["G"]):
        idx = np.nonzero(c["ig"] == i)[0]
        d, e = (sub_orders(p, c, idx, av)[:2]) if idx.size else ([], [])
        d, e = [int(idx[x]) for x in d], [int(idx[x]) for x in e]
        orders.append((idx, d, e))
        do += d; eo += e
        doff.append(len(do)); eoff.append(len(eo))
    p.set_snapshot(av[0], av[1], av[2], np.array(eo, np.int32), np.array(do, np.int32), np.array(eoff, np.int32),
                   np.array(doff, np.int32))
    p.set_schedulable(*sc)
    return av, sc, orders


def queue(seed, c, q):
    rng = np.random.default_rng(seed)
    a = random_apps(rng, q, gpus=seed % 2 == 0)
    a["count"] = np.where(rng.random(q) < 0.1, rng.integers(15, 60, q), a["count"]).astype(np.int32)
    a["young"] = (rng.random(q) < 0.97).astype(np.uint8)
    a["group"] = rng.integers(0, c["G"], q).astype(np.int32)
    return a


def rows(apps, sel):
    return {k: (np.asarray(v)[sel] if v is not None else None) for k, v in apps.items()}


def alone_rows(apps, sel):
    """rows of one instance group for a context holding only its sub-table (one snapshot group: group 0)"""
    r = rows(apps, sel)
    r.pop("group", None)
    return r


def oracle_group(c, av, idx, apps, algo, mode):
    """the literal loop over one instance group: frontend_ref's PotentialNodes on its sub-table, then fitEarlierDrivers"""
    s = sub_table(c, idx)
    d, e = fr.potential_nodes(av[0][idx], av[1][idx], s["zid"], s["nz"], s["rank"], s["cand"], s["unsched"], s["ready"],
                              s["lrd"], s["lre"])
    names = [str(int(v)) for v in idx]
    meta = {names[k]: (int(av[0][v]), int(av[1][v]), int(av[2][v])) for k, v in enumerate(idx)}
    py = [{"drv": (int(apps["drv_cpu"][j]), int(apps["drv_mem"][j]), int(apps["drv_gpu"][j])),
           "exe": (int(apps["exe_cpu"][j]), int(apps["exe_mem"][j]), int(apps["exe_gpu"][j])),
           "count": int(apps["count"][j]), "young": bool(apps["young"][j])} for j in range(len(apps["count"]))]
    _, res = pyref.fit_earlier_drivers(py, [names[k] for k in d], [names[k] for k in e], meta, ALGO_NAME[algo], MODE_NAME[mode])
    return res, meta


@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("G,n,Z,q", [(1, 500, 4, 150), (2, 800, 4, 250), (7, 1500, 5, 500), (140, 6000, 4, 1400)])
def test_fifo_vs_recipe_and_oracle(packer, alone, algo, G, n, Z, q):
    c = groups_case(1800 + G, n, G, Z, empty=(G - 1,) if G > 2 else ())
    apps = queue(1810 + G, c, q)
    for mode in (1, 2):
        label = (G, algo, mode)
        prep(packer, c, orders=False)
        got = packer.pack_batch(apps, algo, mode)
        av, _, orders = host_recipe(alone, c)
        want = alone.pack_batch(apps, algo, mode)
        same_results(got, want, label)
        snap = packer.get_snapshot()
        for x, y in zip(snap, alone.get_snapshot()):
            assert np.array_equal(x, y), label
        drv, exe, off = got
        assert (drv >= 0).any(), label
        for i in range(G):
            sel = np.nonzero(apps["group"] == i)[0]
            idx = orders[i][0]
            if idx.size == 0:
                assert (drv[sel] < 0).all(), label
                continue
            res, meta = oracle_group(c, av, idx, rows(apps, sel), algo, mode)
            for j, (d, ex) in zip(sel, res):
                if d == "unevaluated":
                    assert drv[j] == -2, (label, i, j)
                elif d is None:
                    assert drv[j] == -1, (label, i, j)
                else:
                    assert str(int(drv[j])) == d and [str(int(v)) for v in exe[off[j]:off[j + 1]]] == ex, (label, i, j)
            for k, v in enumerate(idx):
                assert meta[str(int(v))] == (snap[0][v], snap[1][v], snap[2][v]), (label, i, v)


def test_blocked_queue_blocks_only_its_group(packer, alone):
    c = groups_case(1850, 900, 3, 4)
    apps = queue(1851, c, 120)
    apps["young"][:] = 1
    first = [int(np.nonzero(apps["group"] == g)[0][0]) for g in range(3)]
    apps["young"][first[1]] = 0
    apps["drv_cpu"][first[1]] = 1 << 40                   # fits nowhere: instance group 1's queue stops there
    prep(packer, c, orders=False)
    drv, _, _ = packer.pack_batch(apps, 0, 1)
    g1 = apps["group"] == 1
    assert drv[first[1]] == -1 and (drv[g1 & (np.arange(len(drv)) > first[1])] == -2).all()
    assert (drv[~g1] != -2).all() and (drv[~g1] >= 0).any()


def per_sub_table(alone, c, apps, algo, mode=0):
    """every instance group packed on a context holding only its sub-table -> (driver, ExecutorNodes per row) in full indices"""
    drv = np.full(len(apps["count"]), -9, np.int32)
    ex = [None] * len(drv)
    for i in range(c["G"]):
        sel = np.nonzero(apps["group"] == i)[0]
        idx = np.nonzero(c["ig"] == i)[0]
        if sel.size == 0:
            continue
        if idx.size == 0:
            drv[sel] = -1
            continue
        s = sub_table(c, idx)
        alone.prepare_cluster(s["alloc"], s["over"], s["rnode"], s["res"], *sort_args(s))
        d, e, o = alone.pack_batch(alone_rows(apps, sel), algo, mode)
        drv[sel] = np.where(d >= 0, idx[np.maximum(d, 0)], d)
        for k, j in enumerate(sel):
            ex[j] = list(idx[e[o[k]:o[k + 1]]]) if d[k] >= 0 else None
    return drv, ex


@pytest.mark.parametrize("algo", [0, 1, 2])
def test_independent_vs_sub_tables(packer, alone, algo):
    c = groups_case(1900 + algo, 2500, 7, 5, empty=(6,))
    apps = queue(1910 + algo, c, 800)
    prep(packer, c, orders=False)
    drv, exe, off = packer.pack_batch(apps, algo, 0)
    wd, we = per_sub_table(alone, c, apps, algo)
    assert np.array_equal(drv, wd), algo
    for j in np.nonzero(drv >= 0)[0]:
        assert list(exe[off[j]:off[j + 1]]) == we[j], (algo, j)
    assert (drv >= 0).any()


# ---- state rules and refusals -------------------------------------------------------------------------------------------
def _refused(Err, call, status=1, text=None):
    with pytest.raises(Err) as ei:
        call()
    assert ei.value.status == status, str(ei.value)
    if text:
        assert text in str(ei.value), str(ei.value)


def test_snapshot_survives_reservations_and_deltas(packer, alone):
    c = groups_case(1950, 1500, 5, 4)
    apps = queue(1951, c, 300)
    prep(packer, c, orders=False)
    host_recipe(alone, c)
    a, b = packer.pack_batch(apps, 0, 1), alone.pack_batch(apps, 0, 1)
    same_results(a, b, "first")
    packer.reserve_placements(apps, a); alone.reserve_placements(apps, b)
    node = np.array([0, 5, 9], np.int32)
    packer.apply_usage_delta(node, [500] * 3, [GIB] * 3); alone.apply_usage_delta(node, [500] * 3, [GIB] * 3)
    for algo, mode in ((1, 2), (0, 0), (2, 0)):
        same_results(packer.pack_batch(apps, algo, mode), alone.pack_batch(apps, algo, mode), ("after", algo, mode))
    for x, y in zip(packer.get_snapshot(), alone.get_snapshot()):
        assert np.array_equal(x, y)


def test_state_rules_and_refusals(packer, gangpack):
    Err = gangpack.native.GangpackError
    c = groups_case(1960, 900, 3, 4)
    apps = queue(1961, c, 100)
    # the held zone layout is cleared: the layout-from-context forms of the zone entries are refused afterwards
    prepare_groups(packer, c, AZ_AWARE, layout=False)
    packer.pack_fifo_zones_groups(apps, gangpack.native.BP_AZ_AWARE_TIGHTLY_PACK, 1)
    prep(packer, c, orders=False)
    _refused(Err, lambda: packer.pack_fifo_zones_groups(apps, gangpack.native.BP_AZ_AWARE_TIGHTLY_PACK, 1))
    _refused(Err, lambda: packer.pack_fifo_az_aware(apps, 1))
    # bad arguments and a domain refusal: the previous snapshot packs as before
    prep(packer, c, orders=False)
    before = packer.pack_batch(apps, 1, 2)
    prep(packer, c, orders=False)
    snap = packer.get_snapshot()
    bad = c["ig"].copy(); bad[3] = 3
    _refused(Err, lambda: prep(packer, c, ig=bad), text="instance_group")
    bad[3] = -2
    _refused(Err, lambda: prep(packer, c, ig=bad), text="instance_group")
    _refused(Err, lambda: prep(packer, c, G=0), text="n_instance_groups")
    wide = list(sort_args(c)); wide[1] = 1 << 21
    _refused(Err, lambda: packer.prepare_cluster_groups(c["alloc"], c["over"], c["rnode"], c["res"], np.minimum(c["ig"], 1), 2,
                                                        *wide), text="2^22")
    huge = dict(c, alloc=[a.copy() for a in c["alloc"]])
    huge["alloc"][1][0] = 1 << 62
    _refused(Err, lambda: prep(packer, huge), status=6)
    for x, y in zip(snap, packer.get_snapshot()):
        assert np.array_equal(x, y)
    after = packer.pack_batch(apps, 1, 2)
    same_results(after, before, "after refusals")


# ---- packing efficiency per instance group ------------------------------------------------------------------------------
def eff_sub_tables(alone, c, apps, placed, algo, charged, fifo_apps=None):
    """gp_packing_efficiency of each row on a context holding only its instance group's sub-table.  fifo_apps: drain that
    instance group's queue there first (the charged modes), as the full context was drained."""
    drv, exe, off = placed
    out = np.zeros((len(apps["count"]), 4))
    for i in range(c["G"]):
        sel = np.nonzero(apps["group"] == i)[0]
        if sel.size == 0:
            continue
        idx = np.nonzero(c["ig"] == i)[0]
        if idx.size == 0:
            out[sel] = 0.0
            continue
        pos = np.full(len(c["ig"]), -1, np.int32)
        pos[idx] = np.arange(len(idx))
        s = sub_table(c, idx)
        alone.prepare_cluster(s["alloc"], s["over"], s["rnode"], s["res"], *sort_args(s))
        if fifo_apps is not None:
            alone.pack_batch(alone_rows(fifo_apps, np.nonzero(fifo_apps["group"] == i)[0]), algo, charged)
        sub = alone_rows(apps, sel)
        cnt = np.maximum(sub["count"], 0)
        so = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        se = np.concatenate([exe[off[j]:off[j] + cnt[k]] for k, j in enumerate(sel)] + [np.zeros(0, np.int32)])
        sd = np.where(drv[sel] >= 0, pos[np.maximum(drv[sel], 0)], -1).astype(np.int32)
        se = np.where(np.repeat(drv[sel] >= 0, cnt), pos[np.clip(se, 0, len(pos) - 1)], 0).astype(np.int32)
        sub["off"] = so
        out[sel] = alone.packing_efficiency(sub, (sd, se, so), algo, charged)
    return out


def gpu_case(seed, n, G, Z):
    """instance group 1 without GPU nodes, the others with some"""
    c = groups_case(seed, n, G, Z)
    one = c["ig"] == 1
    c["alloc"][2][one] = 0; c["over"][2][one] = 0
    return c


@pytest.mark.parametrize("zones", [False, True])
def test_efficiency_independent(packer, alone, gangpack, zones):
    c = gpu_case(2000, 2000, 5, 4)
    for algo in (0, 1, 2):
        apps = queue(2010 + algo, c, 600)
        prep(packer, c, orders=False)
        placed = packer.pack_batch(apps, algo, 0)
        if zones:                                          # the same availability and SchedulableResources, zone layout
            prepare_groups(packer, c, AZ_AWARE, layout=False)
        got = packer.packing_efficiency_groups(apps, placed, algo, c["ig"], c["G"])
        want = eff_sub_tables(alone, c, apps, placed, algo, 0)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (zones, algo)
        assert (placed[0] >= 0).sum() > 10
        one = (apps["group"] == 1) & (placed[0] >= 0)
        assert (got[one, 2] == 1.0).all() and (got[(apps["group"] == 0) & (placed[0] >= 0), 2] != 1.0).any()


@pytest.mark.parametrize("algo", [0, 1])
def test_efficiency_fifo_charged(packer, alone, algo):
    c = gpu_case(2050, 1500, 4, 4)
    apps = queue(2051 + algo, c, 300)
    for mode in (1, 2):
        prep(packer, c, orders=False)
        placed = packer.pack_batch(apps, algo, mode)
        drv, exe, off = placed
        # one row per instance group: its last placed application, whose usage the drain charged last
        last = [int(np.nonzero((apps["group"] == g) & (drv >= 0))[0][-1]) for g in range(c["G"])]
        one = rows(apps, last)
        cnt = np.maximum(one["count"], 0)
        o = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        e = np.concatenate([exe[off[j]:off[j] + cnt[k]] for k, j in enumerate(last)]).astype(np.int32)
        one["off"] = o
        p1 = (drv[last], e, o)
        got = packer.packing_efficiency_groups(one, p1, algo, c["ig"], c["G"], charged=mode)
        want = eff_sub_tables(alone, c, one, p1, algo, mode, fifo_apps=apps)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (algo, mode)


def test_efficiency_one_group_and_refusals(packer, gangpack):
    Err = gangpack.native.GangpackError
    c = gpu_case(2100, 1200, 3, 4)
    c1 = dict(c, G=1, ig=np.zeros(len(c["ig"]), np.int32))
    apps = queue(2101, c1, 200)
    prep(packer, c1, orders=False)
    placed = packer.pack_batch(apps, 0, 0)
    for algo in (0, 1, 2):
        a = packer.packing_efficiency_groups(apps, placed, algo, c1["ig"], 1)
        b = packer.packing_efficiency(apps, placed, algo)
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), algo
    # refusals on the three-group snapshot
    apps = queue(2102, c, 200)
    prep(packer, c, orders=False)
    drv, exe, off = packer.pack_batch(apps, 0, 0)
    two = [int(j) for j in np.nonzero((apps["group"] == 0) & (drv >= 0))[0][:2]]
    r2 = rows(apps, two)
    cnt = np.maximum(r2["count"], 0)
    o = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    e = np.concatenate([exe[off[j]:off[j] + cnt[k]] for k, j in enumerate(two)]).astype(np.int32)
    r2["off"] = o
    _refused(Err, lambda: packer.packing_efficiency_groups(r2, (drv[two], e, o), 0, c["ig"], 3, charged=1), text="instance group")
    packer.packing_efficiency_groups(r2, (drv[two], e, o), 0, c["ig"], 3)            # independent: fine
    moved = r2.copy(); moved["group"] = np.array([1, 1], np.int32)                  # placed on instance group 0's nodes
    _refused(Err, lambda: packer.packing_efficiency_groups(moved, (drv[two], e, o), 0, c["ig"], 3), text="outside")
    bad = c["ig"].copy(); bad[0] = 3
    _refused(Err, lambda: packer.packing_efficiency_groups(r2, (drv[two], e, o), 0, bad, 3), text="instance_group")
    _refused(Err, lambda: packer.packing_efficiency_groups(r2, (drv[two], e, o), 0, c["ig"], 0))
