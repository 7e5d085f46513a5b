"""CPU model of gp_prepare_cluster_zones_groups (gangpack_sort.cuh, gangpack_zonelayout.cuh), checked against literal
composition: per instance group, pyref.potential_nodes over pyref.node_scheduling_metadata of that instance group's nodes
alone, then test_zone_layout_model.literal_layout, concatenated instance group after instance group.

The device computes every instance group at once:
  1. zone totals and priorities per (instance group, zone) pair: a zone is ranked only against its own instance group's;
  2. one sort by (ig * n_zones + zone priority, memory, cpu, name); nodes in no instance group sort last and are dropped;
  3. the label re-sort by (instance group, label rank, position);
  4. first / has_exec per pair, an exclusive scan of the candidate flags over the driver order, per instance group its
     candidate zones and trailing flag, a scan over the instance groups for each one's first group, the global group of
     every pair, group_rank per node, the partition and the offsets."""
import numpy as np
import pytest

from oracle import pyref
from test_zone_layout_model import AZ_AWARE, BIG, SINGLE_AZ, literal_layout

GIB = 1 << 30


def device_model(c, kind):
    n, G, Z = len(c["ig"]), c["G"], c["Z"]
    ig, zone = c["ig"], c["zone"]
    use = np.zeros((3, n), np.int64)
    for node, r in zip(c["rnode"], c["res"]):
        if 0 <= node < n:
            use[:, node] += r
    avail = c["alloc"] - (use + c["over"])
    tot = {}
    for v in range(n):
        if ig[v] >= 0:
            t = tot.setdefault((ig[v], zone[v]), [0, 0])
            t[0] += int(avail[1, v]); t[1] += int(avail[0, v])
    prio = {}
    for g in range(G):
        zs = sorted(range(Z), key=lambda z: (*tot.get((g, z), (0, 0)), z))
        prio.update({(g, z): p for p, z in enumerate(zs)})
    az = [G * Z if ig[v] < 0 else ig[v] * Z + prio[(ig[v], zone[v])] for v in range(n)]
    order = sorted(range(n), key=lambda v: (az[v], int(avail[1, v]), int(avail[0, v]), c["name_rank"][v]))
    order = [v for v in order if ig[v] >= 0]
    drv = [v for v in order if c["cand"][v]]
    exe = [v for v in order if not c["unsched"][v] and c["ready"][v]]
    lab = lambda rank: (lambda v: (ig[v], BIG if rank[v] < 0 else rank[v]))
    drv = np.array(sorted(drv, key=lab(c["lrd"])), np.int64)            # Python's sort is stable: position breaks ties
    exe = np.array(sorted(exe, key=lab(c["lre"])), np.int64)
    pair = ig * Z + zone
    first = np.full(G * Z, BIG, np.int64)
    np.minimum.at(first, pair[drv], np.arange(len(drv)))
    has = np.zeros(G * Z, bool)
    has[pair[exe]] = True
    flags = (first[pair[drv]] == np.arange(len(drv))) & has[pair[drv]]
    zg = np.full(G * Z, -1, np.int64)
    zg[pair[drv][flags]] = (np.cumsum(flags) - flags)[flags]
    nz = np.bincount(np.nonzero(zg >= 0)[0] // Z, minlength=G)
    trail = np.zeros(G, bool)
    trail[np.nonzero((zg < 0) & ((first != BIG) | has))[0] // Z] = True
    extra = (trail | (nz == 0)) if kind == AZ_AWARE else (nz == 0)
    gbase = np.concatenate([[0], np.cumsum(nz + extra)])
    zbase = np.concatenate([[0], np.cumsum(nz)])
    zone_of_group = np.full(gbase[G], -1, np.int64)
    for p in np.nonzero(zg >= 0)[0]:
        g = p // Z
        zg[p] = zg[p] - zbase[g] + gbase[g]
        zone_of_group[zg[p]] = p % Z
    rank = np.full(n, -9, np.int64)
    for o in (drv, exe):
        r = zg[pair[o]]
        rank[o] = np.where(r >= 0, r, gbase[ig[o]] + nz[ig[o]] if kind == AZ_AWARE else -1)
    out = dict(n_groups=int(gbase[G]), group_off=gbase, n_zones=nz, zone_of_group=zone_of_group, drv=drv, exe=exe)
    for name, o in (("exec", exe), ("drv", drv)):
        key = np.where(rank[o] < 0, BIG, rank[o])
        part = o[np.argsort(key, kind="stable")]
        pr = rank[part]
        off = np.array([int(((pr >= 0) & (pr < g)).sum()) for g in range(gbase[G] + 1)], np.int64)
        out[name + "_off"], out[name + "_order"] = off, part[:off[-1]]
    return out


def literal(c, kind):
    """per instance group: pyref over its own nodes, literal_layout, concatenated"""
    n = len(c["ig"])
    names = ["n%05d" % r for r in c["name_rank"]]
    out = dict(groups=[], drv=[], exe=[], exec_order=[], drv_order=[], exec_off=[0], drv_off=[0], n_zones=[])
    for g in range(c["G"]):
        # nodes in zone-id order first: equal zone totals then rank by zone id, as the library documents
        idx = sorted(np.nonzero(c["ig"] == g)[0], key=lambda v: (c["zone"][v], v))
        res = lambda a, v: tuple(int(a[d][v]) for d in range(3))
        alloc = {names[v]: res(c["alloc"], v) for v in idx}
        over = {names[v]: res(c["over"], v) for v in idx}
        rows = [(names[node], tuple(int(x) for x in r)) for node, r in zip(c["rnode"], c["res"]) if 0 <= node < n and c["ig"][node] == g]
        meta, _ = pyref.node_scheduling_metadata(alloc, over, rows)
        zl = {names[v]: "zone-%d" % c["zone"][v] for v in idx}
        lr = lambda rank: {names[v]: int(rank[v]) for v in idx if rank[v] >= 0}
        d, e = pyref.potential_nodes(meta, zl, [names[v] for v in idx if c["cand"][v]],
                                     unschedulable={names[v] for v in idx if c["unsched"][v]},
                                     not_ready={names[v] for v in idx if not c["ready"][v]},
                                     driver_label_rank=lr(c["lrd"]), exec_label_rank=lr(c["lre"]))
        lay = literal_layout(d, e, zl, kind)
        out["n_zones"].append(lay["n_zones"])
        out["groups"] += lay["zones"]
        out["drv"] += d; out["exe"] += e
        for k in ("exec", "drv"):
            out[k + "_off"] += [len(out[k + "_order"]) + x for x in lay[k + "_off"][1:]]
            out[k + "_order"] += lay[k + "_order"]
    return out, names


def check(c, kind, label):
    got = device_model(c, kind)
    want, names = literal(c, kind)
    assert list(got["n_zones"]) == want["n_zones"], label
    assert got["n_groups"] == len(want["groups"]), label
    assert ["zone-%d" % z if z >= 0 else None for z in got["zone_of_group"]] == want["groups"], label
    assert [names[v] for v in got["drv"]] == want["drv"] and [names[v] for v in got["exe"]] == want["exe"], label
    for k in ("exec", "drv"):
        assert list(got[k + "_off"]) == want[k + "_off"], (label, k)
        assert [names[v] for v in got[k + "_order"]] == want[k + "_order"], (label, k)
    return got


def random_groups_case(rng, n, G, Z, none_p=0.1, empty=(), tie_p=0.0):
    ig = rng.integers(0, G, n)
    ig[rng.random(n) < none_p] = -1
    for e in empty:
        ig[ig == e] = -1
    alloc = np.array([rng.integers(2, 9, n) * 1000, rng.integers(2, 9, n) * GIB, rng.integers(0, 2, n)], np.int64)
    same = rng.random(n) < tie_p                                          # equal (cpu, memory): ties and tied zone totals
    alloc[0][same] = 4000; alloc[1][same] = 4 * GIB
    over = np.array([rng.integers(0, 2, n) * 250, np.zeros(n), np.zeros(n)], np.int64) * (~same)
    R = n
    rnode = np.where(same[np.arange(R) % n], -1, rng.integers(-1, n, R))
    res = np.stack([rng.integers(0, 3, R) * 500, rng.integers(0, 3, R) * (GIB // 2), np.zeros(R, np.int64)], 1)
    return dict(ig=ig, G=G, Z=Z, zone=rng.integers(0, Z, n), alloc=alloc, over=over, rnode=rnode, res=res,
                name_rank=rng.permutation(n), cand=rng.random(n) < 0.7, unsched=rng.random(n) < 0.1, ready=rng.random(n) < 0.9,
                lrd=rng.integers(-1, 3, n), lre=rng.integers(-1, 2, n))


@pytest.mark.parametrize("kind", [SINGLE_AZ, AZ_AWARE])
@pytest.mark.parametrize("G", [1, 2, 7, 140])
def test_segmented_layout_vs_literal_composition(kind, G):
    rng = np.random.default_rng(3000 + 10 * G + kind)
    for t in range(40 if G < 140 else 3):
        n = int(rng.integers(1, 60)) * (1 if G < 140 else 20)
        c = random_groups_case(rng, n, G, int(rng.integers(1, 6)), empty=(G - 1,) if G > 2 and t % 2 else (),
                               tie_p=0.5 if t % 3 == 0 else 0.0)
        if t % 4 == 1:
            c["lrd"][:] = -1; c["lre"][:] = -1                             # no label re-sort
        check(c, kind, (G, t))


@pytest.mark.parametrize("kind", [SINGLE_AZ, AZ_AWARE])
def test_zone_totals_that_tie_and_shared_zone_names(kind):
    """every node equal: every zone total of an instance group ties, so zone ids decide; the same zone ids in every
    instance group rank independently"""
    rng = np.random.default_rng(77)
    for t in range(30):
        c = random_groups_case(rng, 80, 4, 5, tie_p=1.0, none_p=0.0)
        got = check(c, kind, t)
        assert got["n_groups"] >= 4
