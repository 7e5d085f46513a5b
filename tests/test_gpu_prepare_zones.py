"""gp_prepare_cluster_zones: reservations -> availability -> priority orders -> the zone-grouped snapshot of the zone-aware
packers, all on the device.  Checked three ways:
- the layout (zone_of_group, offsets, grouped orders, counts) against the restatement of groupNodesByZone
  (test_zone_layout_model.literal_layout) applied to gp_build_availability -> gp_potential_nodes output;
- the packers' results (single-az-tightly-pack, single-az-minimal-fragmentation, az-aware-tightly-pack; FIFO in both
  accounting modes and independent) against the host recipe it replaces: separate entries, host grouping, gp_set_snapshot +
  gp_set_schedulable and explicit gp_az_orders -- zone, driver node, ExecutorNodes and avg_efficiency bit-identical, and the
  snapshot after FIFO;
- end to end against the literal oracle (node_scheduling_metadata -> Cluster -> potential_nodes -> fifo / binpack)."""
import numpy as np
import pytest

from helpers import random_apps, res_aos
from test_zone_layout_model import AZ_AWARE, SINGLE_AZ, literal_layout

pytestmark = pytest.mark.gpu

ORC = {0: 2, 2: 5, "az": 3}          # device algo -> oracle packer: single-az tightly / minimal-fragmentation, az-aware
G = 1 << 30


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


@pytest.fixture(scope="module")
def recipe(gangpack):
    """a second context for the host recipe, so the two never share state"""
    p = gangpack.GangPacker()
    yield p
    p.close()


def make_case(seed, n, Z, R=None, labels=True, cand_p=0.7, zone_p=None):
    rng = np.random.default_rng(seed)
    names = ["node-%06d" % int(x) for x in rng.permutation(n)]
    alloc = [rng.integers(2, 33, n) * 1000, rng.integers(4, 129, n) * G, (rng.integers(0, 4, n) == 0) * rng.integers(1, 3, n)]
    over = [rng.integers(0, 3, n) * 250, rng.integers(0, 3, n) * (1 << 28), np.zeros(n, np.int64)]
    R = n * 3 if R is None else R
    rnode = rng.integers(-1, n, R).astype(np.int32)
    res = [rng.integers(0, 6, R) * 500, rng.integers(0, 9, R) * (1 << 29), (rng.integers(0, 8, R) == 0).astype(np.int64)]
    p = zone_p if zone_p is not None else rng.random(Z) ** 2 + 0.05
    zone_raw = rng.choice(Z, size=n, p=p / p.sum())
    seen = {}
    zid = np.array([seen.setdefault(int(z), len(seen)) for z in zone_raw], np.int32)    # dense ids in first-seen order
    nz = max(len(seen), 1)
    order = sorted(range(n), key=lambda i: names[i])
    rank = np.empty(n, np.int32); rank[order] = np.arange(n)
    cand = (rng.random(n) < cand_p).astype(np.uint8)
    unsched = (rng.random(n) < 0.1).astype(np.uint8)
    ready = (rng.random(n) < 0.9).astype(np.uint8)
    lrd = rng.integers(-1, 3, n).astype(np.int32) if labels else None          # label ranks that interleave the zones
    lre = rng.integers(-1, 2, n).astype(np.int32) if labels else None
    return dict(names=names, alloc=alloc, over=over, rnode=rnode, res=res, zid=zid, nz=nz, rank=rank, cand=cand,
                unsched=unsched, ready=ready, lrd=lrd, lre=lre)


def sort_args(c):
    return (c["zid"], c["nz"], c["rank"], c["cand"], c["unsched"], c["ready"], c["lrd"], c["lre"])


def prepare(p, c, kind, layout=True):
    return p.prepare_cluster_zones(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c), kind=kind, layout=layout)


def host_recipe(p, c, kind):
    """What a caller does without gp_prepare_cluster_zones: separate entries, grouping on the host, two uploads.
    -> (driver order, executor order, literal layout, schedulable)."""
    av, sc = p.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    d, e = p.potential_nodes(av[0], av[1], *sort_args(c), avail_gpu=av[2])
    ties = p.undefined_ties
    zid = c["zid"] if c["zid"] is not None else np.zeros(len(c["names"]), np.int32)
    lay = literal_layout([int(x) for x in d], [int(x) for x in e], {i: int(z) for i, z in enumerate(zid)}, kind)
    p.set_snapshot(av[0], av[1], av[2], np.array(lay["exec_order"], np.int32), np.array(lay["drv_order"], np.int32),
                   np.array(lay["exec_off"], np.int32), np.array(lay["drv_off"], np.int32))
    p.set_schedulable(*sc)
    return d, e, lay, ties


def check_layout(got, d, e, lay, ties, label):
    assert (got["n_driver"], got["n_executor"]) == (len(d), len(e)), label
    assert got["undefined_ties"] == ties, label
    assert (got["n_zones"], got["n_groups"]) == (lay["n_zones"], lay["n_groups"]), label
    zog = [int(z) if z >= 0 else None for z in got["zone_of_group"][:got["n_groups"]]]
    assert zog == lay["zones"], label
    assert (got["zone_of_group"][got["n_groups"]:] == -1).all(), label
    for k in ("exec_off", "drv_off", "exec_order", "drv_order"):
        assert [int(x) for x in got[k]] == lay[k], (label, k)


def same(a, b, label):
    """(zone, driver_node, executor_nodes, off, avg) of two runs: bit-identical where it is defined."""
    za, da, ea, oa, va = a
    zb, db, eb, ob, vb = b
    assert np.array_equal(oa, ob), label
    bad = np.nonzero((da != db) | ((za != zb) & (da != -2)))[0]
    assert bad.size == 0, (label, bad[:5], za[bad[:5]], zb[bad[:5]], da[bad[:5]], db[bad[:5]])
    for i in np.nonzero(da >= 0)[0]:
        assert np.array_equal(ea[oa[i]:oa[i + 1]], eb[ob[i]:ob[i + 1]]), (label, i)
    placed = da >= 0
    assert np.array_equal(va[placed].view(np.int64), vb[placed].view(np.int64)), label


def apps_for(seed, q, young_p=0.97):
    rng = np.random.default_rng(seed)
    a = random_apps(rng, q, gpus=seed % 2 == 0)
    big = rng.random(q) < 0.1
    a["count"] = np.where(big, rng.integers(20, 90, q), a["count"]).astype(np.int32)
    a["young"] = (rng.random(q) < young_p).astype(np.uint8)
    return a


def run_all(packer, recipe, c, apps, label, fifo_modes=(1, 2)):
    """Every zone-aware packer, FIFO and independent, on the device-prepared snapshot vs the host recipe.  The FIFO kernels
    take at most 64 zones; above that both refuse."""
    for kind in (SINGLE_AZ, AZ_AWARE):
        got = prepare(packer, c, kind)
        d, e, lay, ties = host_recipe(recipe, c, kind)
        check_layout(got, d, e, lay, ties, (label, kind))
        nz = lay["n_zones"]
        if nz > 64:
            with pytest.raises(Exception):
                packer.pack_fifo_az_aware(apps, 1) if kind == AZ_AWARE else packer.pack_fifo_zones(apps, 0, 1)
            fifo_modes = ()
        if kind == SINGLE_AZ:
            for algo in (0, 2):
                same(packer.pack_batch_zones(apps, algo), recipe.pack_batch_zones(apps, algo), (label, "batch", algo))
                for mode in fifo_modes:
                    prepare(packer, c, kind, layout=False)
                    host_recipe(recipe, c, kind)
                    same(packer.pack_fifo_zones(apps, algo, mode), recipe.pack_fifo_zones(apps, algo, mode), (label, "fifo", algo, mode))
                    for x, y in zip(packer.get_snapshot(), recipe.get_snapshot()):
                        assert np.array_equal(x, y), (label, "snapshot", algo, mode)
        else:
            same(packer.pack_batch_az_aware(apps), recipe.pack_batch_az_aware(apps, e, d, nz), (label, "az batch"))
            for mode in fifo_modes:
                prepare(packer, c, kind, layout=False)
                host_recipe(recipe, c, kind)
                same(packer.pack_fifo_az_aware(apps, mode), recipe.pack_fifo_az_aware(apps, mode, e, d, nz), (label, "az fifo", mode))
                for x, y in zip(packer.get_snapshot(), recipe.get_snapshot()):
                    assert np.array_equal(x, y), (label, "az snapshot", mode)


@pytest.mark.parametrize("seed,n,Z", [(1, 30, 1), (2, 120, 3), (3, 400, 7), (4, 1500, 16), (5, 3000, 70), (6, 800, 40), (7, 3000, 5)])
def test_layout_and_packers_vs_host_recipe(packer, recipe, seed, n, Z):
    c = make_case(500 + seed, n, Z, labels=seed != 4)
    apps = apps_for(600 + seed, 300)
    run_all(packer, recipe, c, apps, f"seed {seed}")


def test_one_zone_without_zone_ids(packer, recipe):
    c = make_case(41, 500, 1)
    c["zid"] = None
    apps = apps_for(42, 200)
    got = prepare(packer, c, AZ_AWARE)
    assert got["n_zones"] == 1 and got["zone_of_group"][0] == 0
    run_all(packer, recipe, c, apps, "zone_id NULL")


def test_vs_literal_oracle_end_to_end(oracle, packer):
    """oracle.node_scheduling_metadata -> Cluster(sched, zone labels, unschedulable, ready) -> potential_nodes -> fifo /
    binpack with each zone-aware packer == prepare_cluster_zones -> pack on the device."""
    c = make_case(77, 600, 6)
    apps = apps_for(78, 250)
    names = c["names"]
    n = len(names)
    rn = [names[i] if i >= 0 else "gone" for i in c["rnode"]]
    wav, wsc = oracle.node_scheduling_metadata(names, c["alloc"], c["over"], rn, c["res"])
    labels = ["zone-%d" % z for z in c["zid"]]
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"]); exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    cands = [nm for nm, m in zip(names, c["cand"]) if m]

    def cluster():
        return oracle.Cluster(names, wav[0], wav[1], wav[2], sched=wsc, zone=labels, unschedulable=c["unsched"], ready=c["ready"])
    wd_, we_ = cluster().potential_nodes(cands, c["lrd"], c["lre"])
    for algo, kind, call in ((0, SINGLE_AZ, "zones"), (2, SINGLE_AZ, "zones"), ("az", AZ_AWARE, "az")):
        for mode in (0, 1, 2):
            cl = cluster()
            prepare(packer, c, kind, layout=False)
            if mode == 0:
                wd, we, woff = cl.binpack_batch(ORC[algo], drv, exe, apps["count"], wd_, we_, with_efficiencies=True)
                got = packer.pack_batch_az_aware(apps) if call == "az" else packer.pack_batch_zones(apps, algo)
            else:
                _, wd, we, woff = cl.fifo(ORC[algo], mode, drv, exe, apps["count"], apps["young"], wd_, we_, with_efficiencies=True)
                got = packer.pack_fifo_az_aware(apps, mode) if call == "az" else packer.pack_fifo_zones(apps, algo, mode)
            zone, gd, ge, goff, _ = got
            assert np.array_equal(goff, woff)
            bad = np.nonzero(gd != wd)[0]
            assert bad.size == 0, (algo, mode, bad[:5], gd[bad[:5]], wd[bad[:5]])
            for i in np.nonzero(wd >= 0)[0]:
                assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]]), (algo, mode, i)
            if mode:
                for x, y in zip(packer.get_snapshot(), cl.available()):
                    assert np.array_equal(x, y), (algo, mode)
    assert n == len(wav[0])


def test_no_candidate_zone(packer, recipe, gangpack):
    """Every driver candidate in zone 0, every executor candidate in zone 1: single-AZ gives zone -1 everywhere and FIFO blocks
    with -2 behind; az-aware is gp_pack_batch after plain gp_prepare_cluster."""
    c = make_case(90, 200, 2, zone_p=np.array([0.5, 0.5]), labels=False)
    z = c["zid"]
    first = int(z[0])
    c["cand"] = (z == first).astype(np.uint8)
    c["unsched"] = (z == first).astype(np.uint8)
    c["ready"] = np.ones(200, np.uint8)
    apps = apps_for(91, 120, young_p=0.0)
    got = prepare(packer, c, SINGLE_AZ)
    assert (got["n_zones"], got["n_groups"]) == (0, 1) and len(got["exec_order"]) == 0 and len(got["drv_order"]) == 0
    zone, gd, _, _, _ = packer.pack_batch_zones(apps, 0)
    assert (zone == -1).all() and (gd == -1).all()
    prepare(packer, c, SINGLE_AZ, layout=False)
    zone, gd, _, _, _ = packer.pack_fifo_zones(apps, 0, 1)
    assert (zone == -1).all() and gd[0] == -1 and (gd[1:] == -2).all()
    got = prepare(packer, c, AZ_AWARE)
    assert (got["n_zones"], got["n_groups"]) == (0, 1)
    zone, gd, ge, goff, _ = packer.pack_batch_az_aware(apps)
    packer.prepare_cluster(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c))
    wd, we, woff = packer.pack_batch(apps, 0, 0)
    assert (zone == -1).all() and np.array_equal(gd, wd) and (gd >= 0).any()
    for i in np.nonzero(wd >= 0)[0]:
        assert np.array_equal(ge[goff[i]:goff[i + 1]], we[woff[i]:woff[i + 1]])
    run_all(packer, recipe, c, apps, "no candidate zone")


def test_fallback_reaches_a_driver_only_zone(packer, recipe):
    """The driver's only fitting node lies in a zone without executor candidates: only the trailing group holds it."""
    n = 40
    c = make_case(95, n, 2, R=0, labels=False, zone_p=np.array([0.5, 0.5]))
    z = c["zid"]
    c["alloc"][0][:] = 4000; c["alloc"][1][:] = 8 * G; c["alloc"][2][:] = 0
    only = int(np.nonzero(z == 1)[0][0])
    c["alloc"][0][only] = 64000; c["alloc"][1][only] = 256 * G
    c["unsched"] = (z == 1).astype(np.uint8)                  # zone 1: driver candidates only
    c["ready"] = np.ones(n, np.uint8); c["cand"] = np.ones(n, np.uint8)
    apps = dict(drv_cpu=np.array([32000], np.int64), drv_mem=np.array([128 * G], np.int64), drv_gpu=np.zeros(1, np.int64),
                exe_cpu=np.array([1000], np.int64), exe_mem=np.array([G], np.int64), exe_gpu=np.zeros(1, np.int64),
                count=np.array([3], np.int32), young=np.zeros(1, np.uint8))
    got = prepare(packer, c, AZ_AWARE)
    assert got["n_zones"] == 1 and got["n_groups"] == 2
    zone, gd, _, _, _ = packer.pack_batch_az_aware(apps)
    assert zone[0] == -1 and gd[0] == only
    prepare(packer, c, AZ_AWARE, layout=False)
    zone, gd, _, _, _ = packer.pack_fifo_az_aware(apps, 1)
    assert zone[0] == -1 and gd[0] == only
    run_all(packer, recipe, c, apps, "driver-only zone")


def _zones_case(seed, n, Z):
    """n nodes spread over exactly Z zones, each with driver and executor candidates"""
    c = make_case(seed, n, Z, labels=False, zone_p=np.ones(Z))
    c["cand"] = np.ones(n, np.uint8); c["unsched"] = np.zeros(n, np.uint8); c["ready"] = np.ones(n, np.uint8)
    return c


@pytest.mark.parametrize("Z", [64, 65, 70])
def test_zone_bounds(packer, recipe, gangpack, Z):
    c = _zones_case(130 + Z, 20 * Z, Z)
    apps = apps_for(131, 150)
    got = prepare(packer, c, AZ_AWARE)
    assert got["n_zones"] == Z
    d, e, lay, _ = host_recipe(recipe, c, AZ_AWARE)
    same(packer.pack_batch_az_aware(apps), recipe.pack_batch_az_aware(apps, e, d, Z), ("batch", Z))
    if Z <= 64:
        prepare(packer, c, AZ_AWARE, layout=False)
        host_recipe(recipe, c, AZ_AWARE)
        same(packer.pack_fifo_az_aware(apps, 2), recipe.pack_fifo_az_aware(apps, 2, e, d, Z), ("fifo", Z))
    else:
        with pytest.raises(gangpack.native.GangpackError) as ei:
            packer.pack_fifo_az_aware(apps, 1)
        assert ei.value.status == 1 and "0..64" in str(ei.value)


def test_large_cluster_with_a_long_queue(packer, recipe):
    """50 000 nodes in 16 zones, 10 000 queued drivers, 100 000 reservations."""
    c = make_case(160, 50000, 16, R=100000)
    apps = apps_for(161, 10000)
    run_all(packer, recipe, c, apps, "50k", fifo_modes=(1,))


def test_refusals_and_state(packer, recipe, gangpack):
    Err = gangpack.native.GangpackError
    c = make_case(170, 300, 4)
    apps = apps_for(171, 50)
    # NULL orders after a snapshot from gp_set_snapshot / gp_prepare_cluster: refused as before
    d, e, lay, _ = host_recipe(packer, c, AZ_AWARE)
    for call in (lambda: packer.pack_batch_az_aware(apps), lambda: packer.pack_fifo_az_aware(apps, 1)):
        with pytest.raises(Err) as ei:
            call()
        assert ei.value.status == 1
    packer.prepare_cluster(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c))
    with pytest.raises(Err) as ei:
        packer.pack_batch_az_aware(apps)
    assert ei.value.status == 1
    # NULL after a single-AZ layout
    prepare(packer, c, SINGLE_AZ)
    for call in (lambda: packer.pack_batch_az_aware(apps), lambda: packer.pack_fifo_az_aware(apps, 1)):
        with pytest.raises(Err) as ei:
            call()
        assert ei.value.status == 1 and "GP_LAYOUT_SINGLE_AZ" in str(ei.value)
    # explicit orders after a device-built layout: no host copy to check them against
    got = prepare(packer, c, AZ_AWARE)
    with pytest.raises(Err) as ei:
        packer.pack_batch_az_aware(apps, e, d, got["n_zones"])
    assert ei.value.status == 1
    # a bad kind
    with pytest.raises(Err) as ei:
        prepare(packer, c, 7)
    assert ei.value.status == 1
    # gp_prepare_cluster_zones -> gp_set_snapshot -> NULL orders: refused again
    prepare(packer, c, AZ_AWARE)
    packer.set_snapshot(*packer.get_snapshot(), np.array(lay["exec_order"], np.int32), np.array(lay["drv_order"], np.int32),
                        np.array(lay["exec_off"], np.int32), np.array(lay["drv_off"], np.int32))
    with pytest.raises(Err):
        packer.pack_fifo_az_aware(apps, 1)
    # the layout survives gp_reserve_placements(subtract) and gp_apply_usage_delta
    prepare(packer, c, AZ_AWARE)
    host_recipe(recipe, c, AZ_AWARE)
    zone, gd, ge, goff, _ = packer.pack_batch_az_aware(apps)
    zone2, gd2, ge2, goff2, _ = recipe.pack_batch_az_aware(apps, e, d, lay["n_zones"])
    packer.reserve_placements(apps, (gd, ge, goff)); recipe.reserve_placements(apps, (gd2, ge2, goff2))
    packer.apply_usage_delta(np.array([0, 1], np.int32), [500, 500], [G, G]); recipe.apply_usage_delta(np.array([0, 1], np.int32), [500, 500], [G, G])
    same(packer.pack_fifo_az_aware(apps, 1), recipe.pack_fifo_az_aware(apps, 1, e, d, lay["n_zones"]), "after reservations")


def test_arena_reuse_and_an_interleaved_sort(packer, recipe):
    """A smaller call after a larger one, and a gp_potential_nodes call between the layout and the pack."""
    big, small = make_case(180, 4000, 12), make_case(181, 150, 3)
    apps = apps_for(182, 200)
    prepare(packer, big, AZ_AWARE)
    run_all(packer, recipe, small, apps, "small after big", fifo_modes=(2,))
    prepare(packer, small, AZ_AWARE)
    d, e, lay, _ = host_recipe(recipe, small, AZ_AWARE)
    packer.potential_nodes(*[np.arange(4000, dtype=np.int64)] * 2)           # reuses the sort's scratch
    same(packer.pack_fifo_az_aware(apps, 1), recipe.pack_fifo_az_aware(apps, 1, e, d, lay["n_zones"]), "sort in between")
