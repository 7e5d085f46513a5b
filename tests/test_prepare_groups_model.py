"""CPU-only model of gp_prepare_cluster_groups' composition: one instance-group-major PotentialNodes pass (the instance
group leads the sort key, zone priority per (instance group, zone), the label re-sort keyed by (instance group, rank,
position)), then each instance group's range found by binary search (gp_ig_offsets) -- against PotentialNodes run
literally (pyref) over every instance group's nodes alone and concatenated.  Covers 1, 2, 7 and 140 instance groups,
empty ones, nodes in none, label re-sorts, shared zone names with tied totals, and an instance group above the 4 096-key
sort tile."""
import numpy as np
import pytest

from oracle import pyref
from test_zone_layout_groups_model import device_model, random_groups_case
from test_zone_layout_model import SINGLE_AZ


def model(c):
    """-> (driver order, executor order, drv_off, exec_off) of the one instance-group-major pass"""
    m = device_model(c, SINGLE_AZ)
    ig = c["ig"]
    offs = []
    for o in (m["drv"], m["exe"]):
        assert (np.diff(ig[o]) >= 0).all()                                 # instance-group-major
        offs.append(np.searchsorted(ig[o], np.arange(c["G"] + 1), side="left"))
    return m["drv"], m["exe"], offs[0], offs[1]


def literal(c):
    """PotentialNodes per instance group over its own nodes (pyref), concatenated, with the CSR offsets"""
    n = len(c["ig"])
    names = ["n%05d" % r for r in c["name_rank"]]
    drv, exe, doff, eoff = [], [], [0], [0]
    for g in range(c["G"]):
        idx = sorted(np.nonzero(c["ig"] == g)[0], key=lambda v: (c["zone"][v], v))
        res = lambda a, v: tuple(int(a[d][v]) for d in range(3))
        alloc = {names[v]: res(c["alloc"], v) for v in idx}
        over = {names[v]: res(c["over"], v) for v in idx}
        rows = [(names[node], tuple(int(x) for x in r)) for node, r in zip(c["rnode"], c["res"]) if 0 <= node < n and c["ig"][node] == g]
        meta, _ = pyref.node_scheduling_metadata(alloc, over, rows)
        lr = lambda rank: {names[v]: int(rank[v]) for v in idx if rank[v] >= 0}
        d, e = pyref.potential_nodes(meta, {names[v]: "zone-%d" % c["zone"][v] for v in idx}, [names[v] for v in idx if c["cand"][v]],
                                     unschedulable={names[v] for v in idx if c["unsched"][v]},
                                     not_ready={names[v] for v in idx if not c["ready"][v]},
                                     driver_label_rank=lr(c["lrd"]), exec_label_rank=lr(c["lre"]))
        drv += d; exe += e
        doff.append(len(drv)); eoff.append(len(exe))
    return drv, exe, doff, eoff, names


def check(c, label):
    d, e, doff, eoff = model(c)
    wd, we, wdoff, weoff, names = literal(c)
    assert [names[v] for v in d] == wd and [names[v] for v in e] == we, label
    assert list(doff) == wdoff and list(eoff) == weoff, label


@pytest.mark.parametrize("G", [1, 2, 7, 140])
def test_instance_group_major_vs_literal(G):
    rng = np.random.default_rng(5000 + G)
    for t in range(30 if G < 140 else 3):
        n = int(rng.integers(1, 60)) * (1 if G < 140 else 20)
        c = random_groups_case(rng, n, G, int(rng.integers(1, 6)), empty=(G - 1,) if G > 2 and t % 2 else (),
                               tie_p=0.5 if t % 3 == 0 else 0.0)
        if t % 4 == 1:
            c["lrd"][:] = -1; c["lre"][:] = -1                             # no label re-sort
        check(c, (G, t))


def test_tied_zone_totals_and_shared_zone_names():
    rng = np.random.default_rng(77)
    for t in range(20):
        check(random_groups_case(rng, 80, 4, 5, tie_p=1.0, none_p=0.0), t)


def test_instance_group_above_the_sort_tile():
    rng = np.random.default_rng(91)
    c = random_groups_case(rng, 9000, 2, 3, none_p=0.02)
    assert min((c["ig"] == 0).sum(), (c["ig"] == 1).sum()) > 4096
    check(c, "tile")
