"""gp_prepare_cluster_zones_groups: reservations -> availability -> PotentialNodes per instance group -> every instance
group's zone-grouped layout, on the device, then gp_pack_fifo_zones_groups(groups == NULL) from it.  Checked:
- layout identity: each instance group's slice (groups, zone_of_group, offsets, grouped and undivided orders, counts,
  undefined ties) equals gp_prepare_cluster_zones / gp_potential_nodes on a second context holding only that instance
  group's sub-table, mapped back to full-table indices; instance_group = NULL equals gp_prepare_cluster_zones outright;
- FIFO bit for bit, all three zone-aware packers in both FIFO modes, against the host recipe feeding the explicit layout
  (gp_build_availability -> gp_potential_nodes per instance group -> host grouping -> gp_set_snapshot + gp_instance_groups)
  and, per instance group, against the literal oracle's loop;
- the state rules: what keeps the held layout, what replaces it, and what is refused."""
import numpy as np
import pytest

from helpers import random_apps
from test_gpu_prepare_zones import G as GIB, make_case, sort_args
from test_gpu_zone_fifo_groups import AZ_AWARE as BP_AZ, SINGLE_MINFRAG, SINGLE_TIGHT, Case, expected
from test_zone_layout_model import AZ_AWARE, SINGLE_AZ

pytestmark = pytest.mark.gpu

PACKERS = [SINGLE_TIGHT, SINGLE_MINFRAG, BP_AZ]
KIND = {SINGLE_TIGHT: SINGLE_AZ, SINGLE_MINFRAG: SINGLE_AZ, BP_AZ: AZ_AWARE}


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


@pytest.fixture(scope="module")
def alone(gangpack):
    """a second context: one instance group's sub-table at a time, or the host recipe"""
    p = gangpack.GangPacker()
    yield p
    p.close()


def groups_case(seed, n, G, Z, labels=True, none_p=0.1, empty=()):
    """make_case's node table (zone ids shared by name across instance groups) with an instance group per node:
    some nodes in none, the instance groups in `empty` without nodes."""
    c = make_case(seed, n, Z, labels=labels)
    rng = np.random.default_rng(seed + 7)
    ig = rng.integers(0, G, n).astype(np.int32)
    ig[rng.random(n) < none_p] = -1
    for e in empty:
        ig[ig == e] = -1
    c["ig"], c["G"] = ig, G
    return c


_CASE = object()


def prepare_groups(p, c, kind, layout=True, ig=_CASE):
    return p.prepare_cluster_zones_groups(c["alloc"], c["over"], c["rnode"], c["res"], c["ig"] if ig is _CASE else ig, c["G"],
                                          *sort_args(c), kind=kind, layout=layout)


def sub_table(c, idx):
    """instance group sub-table: its nodes, their reservations (others dropped), name ranks renumbered"""
    pos = np.full(len(c["names"]), -1, np.int64)
    pos[idx] = np.arange(len(idx))
    rn = np.where(c["rnode"] >= 0, pos[np.maximum(c["rnode"], 0)], -1).astype(np.int32)
    rank = np.empty(len(idx), np.int32)
    rank[np.argsort(c["rank"][idx], kind="stable")] = np.arange(len(idx))
    s = dict(alloc=[a[idx] for a in c["alloc"]], over=[o[idx] for o in c["over"]], rnode=rn, res=c["res"],
             zid=c["zid"][idx] if c["zid"] is not None else None, nz=c["nz"], rank=rank, names=[c["names"][i] for i in idx])
    for k in ("cand", "unsched", "ready", "lrd", "lre"):
        s[k] = c[k][idx] if c[k] is not None else None
    return s


def check_identity(packer, alone, c, kind, label):
    got = prepare_groups(packer, c, kind)
    G = c["G"]
    goff = got["group_off"]
    assert goff[0] == 0 and goff[G] == got["n_groups"], label
    tot_ties = 0
    for i in range(G):
        idx = np.nonzero(c["ig"] == i)[0]
        g0, g1 = int(goff[i]), int(goff[i + 1])
        e0, e1, d0, d1 = (int(x) for x in (got["exec_off"][i], got["exec_off"][i + 1], got["drv_off"][i], got["drv_off"][i + 1]))
        if idx.size == 0:               # the layout of "no candidate zone" over empty orders
            assert got["n_zones"][i] == 0 and g1 - g0 == 1 and got["zone_of_group"][g0] == -1, (label, i)
            assert e1 == e0 and d1 == d0 and got["ig_undefined_ties"][i] == 0, (label, i)
            assert got["group_exec_off"][g1] == got["group_exec_off"][g0] and got["group_drv_off"][g1] == got["group_drv_off"][g0]
            continue
        s = sub_table(c, idx)
        want = alone.prepare_cluster_zones(s["alloc"], s["over"], s["rnode"], s["res"], *sort_args(s), kind=kind)
        av, _ = alone.build_availability(s["alloc"], s["over"], s["rnode"], s["res"])
        d, e = alone.potential_nodes(av[0], av[1], *sort_args(s), avail_gpu=av[2])
        assert want["undefined_ties"] == alone.undefined_ties
        lab = (label, i)
        assert got["n_zones"][i] == want["n_zones"] and g1 - g0 == want["n_groups"], lab
        assert list(got["zone_of_group"][g0:g1]) == list(want["zone_of_group"][:want["n_groups"]]), lab
        assert got["ig_undefined_ties"][i] == want["undefined_ties"], lab
        tot_ties += want["undefined_ties"]
        assert list(got["exec_order"][e0:e1]) == list(idx[e]) and list(got["drv_order"][d0:d1]) == list(idx[d]), lab
        assert (e1 - e0, d1 - d0) == (want["n_executor"], want["n_driver"]), lab
        for k in ("exec", "drv"):
            off = got["group_%s_off" % k][g0:g1 + 1]
            assert list(off - off[0]) == list(want["%s_off" % k]), (lab, k)
            assert list(got["group_%s_order" % k][off[0]:off[-1]]) == list(idx[want["%s_order" % k]]), (lab, k)
    assert got["undefined_ties"] == tot_ties and got["ig_undefined_ties"].sum() == tot_ties, label
    assert got["n_driver"] == got["drv_off"][G] and got["n_executor"] == got["exec_off"][G], label
    return got


@pytest.mark.parametrize("G,n,Z", [(1, 400, 5), (2, 600, 4), (7, 1500, 9), (140, 4000, 6)])
def test_layout_identity(packer, alone, G, n, Z):
    c = groups_case(700 + G, n, G, Z, empty=(G - 1,) if G > 2 else ())
    for kind in (SINGLE_AZ, AZ_AWARE):
        check_identity(packer, alone, c, kind, (G, kind))


def test_identity_edges(packer, alone):
    """an instance group without a candidate zone, one with 65 candidate zones, GPU nodes whose ties the reference leaves
    undefined, and no label ranks"""
    c = groups_case(720, 3000, 4, 70, labels=False, none_p=0.05)
    n = len(c["names"])
    ig, z = c["ig"], c["zid"]
    c["nz"] = 70
    c["cand"] = np.ones(n, np.uint8); c["unsched"] = np.zeros(n, np.uint8); c["ready"] = np.ones(n, np.uint8)
    # instance group 0: one node per zone id 0..69 and more (70 zones, 65+ of them candidates)
    zero = np.nonzero(ig == 0)[0]
    z[zero] = np.arange(len(zero)) % 70
    # instance group 1: drivers only in zone 0, executors only elsewhere: no candidate zone
    one = np.nonzero(ig == 1)[0]
    c["cand"][one] = (z[one] == 0).astype(np.uint8)
    c["unsched"][one] = (z[one] == 0).astype(np.uint8)
    # instance group 2: equal memory and cpu, different gpu -> undefined ties
    two = np.nonzero(ig == 2)[0]
    c["alloc"][0][two] = 8000; c["alloc"][1][two] = 32 * GIB; c["alloc"][2][two] = np.arange(len(two)) % 3
    c["over"][0][two] = 0; c["over"][1][two] = 0
    c["rnode"][np.isin(c["rnode"], two)] = -1
    for kind in (SINGLE_AZ, AZ_AWARE):
        got = check_identity(packer, alone, c, kind, ("edges", kind))
        assert got["n_zones"][0] >= 65 and got["n_zones"][1] == 0 and got["ig_undefined_ties"][2] > 0


def test_null_instance_group_is_prepare_cluster_zones(packer, alone):
    c = groups_case(730, 1200, 1, 6)
    for kind in (SINGLE_AZ, AZ_AWARE):
        got = prepare_groups(packer, c, kind, ig=None)
        want = alone.prepare_cluster_zones(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c), kind=kind)
        assert got["n_groups"] == want["n_groups"] and got["n_zones"][0] == want["n_zones"]
        assert got["undefined_ties"] == want["undefined_ties"] == got["ig_undefined_ties"][0]
        assert list(got["zone_of_group"]) == list(want["zone_of_group"][:want["n_groups"]])
        for k in ("exec", "drv"):
            assert list(got["group_%s_off" % k]) == list(want["%s_off" % k])
            assert list(got["group_%s_order" % k]) == list(want["%s_order" % k])
        for x, y in zip(packer.get_snapshot(), alone.get_snapshot()):
            assert np.array_equal(x, y)


# ---- FIFO from the held layout -------------------------------------------------------------------------------------------
def recipe(p, c):
    """The host recipe: availability, PotentialNodes per instance group on its sub-table, grouping on the host (Case of
    test_gpu_zone_fifo_groups), then the explicit layout.  -> Case"""
    av, sc = p.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    orders = []
    for i in range(c["G"]):
        idx = np.nonzero(c["ig"] == i)[0]
        if idx.size == 0:
            orders.append(([], []))
            continue
        s = sub_table(c, idx)
        d, e = p.potential_nodes(av[0][idx], av[1][idx], *sort_args(s), avail_gpu=av[2][idx])
        orders.append(([int(idx[x]) for x in d], [int(idx[x]) for x in e]))
    case = Case.__new__(Case)
    case.G, case.n = c["G"], len(c["names"])
    case.cpu, case.mem, case.gpu = av
    case.sc, case.sm, case.sg = sc
    case.zone_of = np.asarray(c["zid"], np.int64) if c["zid"] is not None else np.zeros(case.n, np.int64)
    case.orders, case.names = orders, c["names"]
    case.labels = ["z%d" % z for z in case.zone_of]
    return case


def fifo_apps(seed, c, q):
    rng = np.random.default_rng(seed)
    a = random_apps(rng, q, gpus=seed % 2 == 0)
    a["count"] = np.where(rng.random(q) < 0.1, rng.integers(15, 60, q), a["count"]).astype(np.int32)
    a["young"] = (rng.random(q) < 0.97).astype(np.uint8)
    a["group"] = rng.integers(0, c["G"], q).astype(np.int32)
    return a


def same_fifo(a, b, sa, sb, label):
    (za, da, ea, oa, va), (zb, db, eb, ob, vb) = a, b
    assert np.array_equal(oa, ob) and np.array_equal(da, db), (label, np.nonzero(da != db)[0][:5])
    placed = da >= 0
    assert np.array_equal(za[placed], zb[placed]), label
    for j in np.nonzero(placed)[0]:
        assert np.array_equal(ea[oa[j]:oa[j + 1]], eb[ob[j]:ob[j + 1]]), (label, j)
    assert np.array_equal(va.view(np.uint64), vb.view(np.uint64)), label
    for x, y in zip(sa, sb):
        assert np.array_equal(x, y), label


def held_vs_recipe(packer, alone, c, apps, packer_id, mode, label):
    prepare_groups(packer, c, KIND[packer_id], layout=False)
    case = recipe(alone, c)
    kw, per = case.load(alone, packer_id == BP_AZ)
    got = packer.pack_fifo_zones_groups(apps, packer_id, mode)
    gst = packer.stats()
    want = alone.pack_fifo_zones_groups(apps, packer_id, mode, **kw)
    wst = alone.stats()
    same_fifo(got, want, packer.get_snapshot(), alone.get_snapshot(), label)
    for k in ("nodes_scanned", "drivers_tried", "scan_path_apps"):
        assert gst[k] == wst[k], (label, k)
    return case, per, got, gst


@pytest.mark.parametrize("packer_id", PACKERS)
@pytest.mark.parametrize("G,n,Z,q", [(1, 500, 4, 150), (2, 800, 4, 250), (7, 1500, 5, 500), (140, 6000, 4, 1400)])
def test_fifo_vs_recipe_and_oracle(oracle, packer, alone, packer_id, G, n, Z, q):
    c = groups_case(800 + G, n, G, Z, empty=(G - 1,) if G > 2 else ())
    apps = fifo_apps(810 + G, c, q)
    for mode in (1, 2):
        label = (G, packer_id, mode)
        case, per, got, gst = held_vs_recipe(packer, alone, c, apps, packer_id, mode, label)
        wz, wd, we, wavg, wavail, wst = expected(case, alone, oracle, apps, packer_id, mode, per)
        zone, drv, ge, goff, avg = got
        assert np.array_equal(drv, wd), label
        placed = wd >= 0
        assert np.array_equal(zone[placed], wz[placed]), label
        for j in np.nonzero(placed)[0]:
            assert list(ge[goff[j]:goff[j + 1]]) == we[j], (label, j)
        assert np.array_equal(avg.view(np.uint64), wavg.view(np.uint64)), label
        for x, y in zip(packer.get_snapshot(), wavail):
            assert np.array_equal(x, y), label
        for k in wst:
            assert gst[k] == wst[k], (label, k, gst[k], wst[k])
        assert (drv >= 0).any(), label


def test_held_layout_survives_reservations_and_deltas(packer, alone):
    c = groups_case(900, 1500, 5, 4)
    apps = fifo_apps(901, c, 300)
    for packer_id in (SINGLE_TIGHT, BP_AZ):
        prepare_groups(packer, c, KIND[packer_id], layout=False)
        case = recipe(alone, c)
        kw, _ = case.load(alone, packer_id == BP_AZ)
        a = packer.pack_fifo_zones_groups(apps, packer_id, 1)
        b = alone.pack_fifo_zones_groups(apps, packer_id, 1, **kw)
        same_fifo(a, b, packer.get_snapshot(), alone.get_snapshot(), "first")
        packer.reserve_placements(apps, a[1:4]); alone.reserve_placements(apps, b[1:4])
        node = np.array([0, 5, 9], np.int32)
        packer.apply_usage_delta(node, [500] * 3, [GIB] * 3); alone.apply_usage_delta(node, [500] * 3, [GIB] * 3)
        same_fifo(packer.pack_fifo_zones_groups(apps, packer_id, 2), alone.pack_fifo_zones_groups(apps, packer_id, 2, **kw),
                  packer.get_snapshot(), alone.get_snapshot(), ("after reservations", packer_id))


def _refused(Err, call, text=None):
    with pytest.raises(Err) as ei:
        call()
    assert ei.value.status == 1, str(ei.value)
    if text:
        assert text in str(ei.value), str(ei.value)


def test_state_rules_and_refusals(packer, gangpack):
    Err = gangpack.native.GangpackError
    c = groups_case(910, 900, 3, 4)
    apps = fifo_apps(911, c, 100)
    held = lambda pid=SINGLE_TIGHT: packer.pack_fifo_zones_groups(apps, pid, 1)
    # each of the four other snapshot-setting calls replaces the held layout
    av, sc = packer.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    d, e = packer.potential_nodes(av[0], av[1], *sort_args(c))
    import torch
    dev = [torch.as_tensor(np.asarray(x), dtype=dt, device="cuda") for x, dt in
           ((av[0], torch.int64), (av[1], torch.int64), (av[2], torch.int64), ([0, len(e)], torch.int32), (e, torch.int32),
            ([0, len(d)], torch.int32), (d, torch.int32))]
    setters = [lambda: packer.set_snapshot(av[0], av[1], av[2], e, d),
               lambda: (packer.set_snapshot_device(*dev), packer.synchronize()),
               lambda: packer.prepare_cluster(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c)),
               lambda: packer.prepare_cluster_zones(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c), kind=SINGLE_AZ)]
    for s in setters:
        prepare_groups(packer, c, SINGLE_AZ, layout=False)
        held()
        s()
        packer.set_schedulable(*sc)
        _refused(Err, held, "gp_prepare_cluster_zones_groups")
    # packer / kind mismatch
    prepare_groups(packer, c, SINGLE_AZ, layout=False)
    _refused(Err, lambda: held(BP_AZ), "GP_LAYOUT_AZ_AWARE")
    prepare_groups(packer, c, AZ_AWARE, layout=False)
    _refused(Err, lambda: held(SINGLE_MINFRAG), "GP_LAYOUT_SINGLE_AZ")
    # explicit groups after the device-built layout: no host copy, as before
    _refused(Err, lambda: packer.pack_fifo_zones_groups(apps, BP_AZ, 1, group_off=[0, 1, 2, 3]), "laid out by gp_set_snapshot")
    # the single-instance-group zone entries after a multi-group prepare
    single = [lambda: packer.pack_fifo_zones(apps, 0, 1), lambda: packer.pack_batch_zones(apps, 0),
              lambda: packer.pack_fifo_az_aware(apps, 1), lambda: packer.pack_batch_az_aware(apps)]
    for kind in (SINGLE_AZ, AZ_AWARE):
        prepare_groups(packer, c, kind, layout=False)
        for call in single:
            _refused(Err, call, "gp_pack_fifo_zones_groups")
    # ... but not after a one-group prepare, which leaves the context as gp_prepare_cluster_zones does
    c1 = dict(c, G=1, ig=np.where(c["ig"] >= 0, 0, -1).astype(np.int32))
    prepare_groups(packer, c1, AZ_AWARE, layout=False)
    packer.pack_fifo_az_aware(apps, 1)
    # more than 64 candidate zones: prepared, refused at FIFO time
    big = groups_case(920, 3000, 2, 70, labels=False, none_p=0.0)
    big["nz"] = 70
    big["cand"][:] = 1; big["unsched"][:] = 0; big["ready"][:] = 1
    big["zid"][big["ig"] == 0] = np.arange(int((big["ig"] == 0).sum())) % 70
    for kind, pid in ((SINGLE_AZ, SINGLE_TIGHT), (AZ_AWARE, BP_AZ)):
        got = prepare_groups(packer, big, kind, layout=False)
        assert got["n_zones"][0] > 64
        _refused(Err, lambda: held(pid), "more than 64")
    # bad arguments, and a domain refusal: the previous layout stays usable with identical results
    prepare_groups(packer, c, AZ_AWARE, layout=False)
    before = held(BP_AZ)
    snap = packer.get_snapshot()
    prepare_groups(packer, c, AZ_AWARE, layout=False)
    bad_ig = c["ig"].copy(); bad_ig[3] = 3
    _refused(Err, lambda: prepare_groups(packer, c, AZ_AWARE, ig=bad_ig), "instance_group")
    bad_ig[3] = -2
    _refused(Err, lambda: prepare_groups(packer, c, AZ_AWARE, ig=bad_ig), "instance_group")
    _refused(Err, lambda: packer.prepare_cluster_zones_groups(c["alloc"], c["over"], c["rnode"], c["res"], c["ig"], 0, *sort_args(c)))
    # more than 2^22 (instance group, zone) pairs with several instance groups
    wide = list(sort_args(c)); wide[1] = 1 << 21
    _refused(Err, lambda: packer.prepare_cluster_zones_groups(c["alloc"], c["over"], c["rnode"], c["res"], np.minimum(c["ig"], 1), 2,
                                                              *wide, kind=AZ_AWARE), "2^22")
    huge = dict(c, alloc=[a.copy() for a in c["alloc"]])
    huge["alloc"][1][0] = 1 << 62
    with pytest.raises(Err) as ei:
        prepare_groups(packer, huge, AZ_AWARE)
    assert ei.value.status == 6
    after = held(BP_AZ)
    for x, y in zip(before, after):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    for x, y in zip(snap, packer.get_snapshot()):
        assert np.array_equal(x, y)
