"""CPU model of gp_prepare_cluster_zones' grouping (gangpack_zonelayout.cuh), checked against a literal groupNodesByZone.

The device groups the two undivided priority orders by zone without sorting the zones:
  1. first[z] = smallest driver-order position of a node of zone z (atomicMin), has_exec[z] = z holds an executor candidate;
  2. driver position i is flagged when first[zone] == i and has_exec[zone]; an exclusive scan of the flags numbers the
     candidate zones, in the order of their first appearance in the driver order;
  3. group_rank[node] = its zone's number, n_zones for the trailing group (az-aware) or -1 (dropped, single-AZ);
  4. a stable re-sort of each order by group_rank (the label re-sort: -1 sorts last) partitions it;
  5. off[g] = number of positions whose rank is below g, for every g up to the bound sort->n_zones + 1.
This file restates those steps in numpy and compares them with the literal statement of the host layer
(binpack::ZoneGroups / AzAwareLayout: single_az.go:30-41,57-73, az_aware_pack_tightly.go:27-38) on thousands of orders.
It also checks the ctypes mirror of gp_zone_layout against a C compiler."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SINGLE_AZ, AZ_AWARE = 0, 1
BIG = 0x7FFFFFFF


def device_model(drv, exe, zone, n_zone_ids, kind):
    """The device algorithm on index arrays.  zone: [n_nodes] zone id per node.  -> dict like the layout the call returns,
    plus `bound_off` (the offsets up to the bound, which the slot layout reads)."""
    drv, exe, zone = np.asarray(drv, np.int64), np.asarray(exe, np.int64), np.asarray(zone, np.int64)
    Z = n_zone_ids
    first = np.full(Z, BIG, np.int64)
    np.minimum.at(first, zone[drv], np.arange(len(drv)))
    has_exec = np.zeros(Z, bool)
    has_exec[zone[exe]] = True
    dz = zone[drv]
    flags = (first[dz] == np.arange(len(drv))) & has_exec[dz]
    excl = np.cumsum(flags) - flags
    nz = int(flags.sum())
    zone_group = np.full(Z, -1, np.int64)
    zone_group[dz[flags]] = excl[flags]
    zone_of_group = np.full(Z + 1, -1, np.int64)
    zone_of_group[excl[flags]] = dz[flags]
    group_rank = np.full(len(zone), -9, np.int64)
    trailing = False
    for order in (drv, exe):
        r = zone_group[zone[order]]
        trailing |= bool((r < 0).any())
        group_rank[order] = np.where(r < 0, nz if kind == AZ_AWARE else -1, r)
    n_groups = (nz + (1 if (trailing or nz == 0) else 0)) if kind == AZ_AWARE else max(nz, 1)
    g_bound = Z + 1
    out = dict(n_zones=nz, n_groups=n_groups, zone_of_group=zone_of_group)
    for name, order in (("exec", exe), ("drv", drv)):
        r = group_rank[order]
        key = np.where(r < 0, BIG, r)
        part = order[np.argsort(key, kind="stable")]            # the label re-sort: (rank, position) ascending
        pr = group_rank[part]
        eff = np.where(pr < 0, BIG, pr)
        assert (np.diff(eff) >= 0).all()
        off = np.array([int(((pr >= 0) & (pr < g)).sum()) for g in range(g_bound + 1)], np.int64)
        assert (np.searchsorted(eff, np.arange(g_bound + 1), side="left") == off).all()    # the kernel's binary search
        out[name + "_bound_off"] = off
        out[name + "_off"] = off[:n_groups + 1]
        out[name + "_order"] = part[:off[g_bound]]
    return out


def literal_layout(drv, exe, zone_label, kind):
    """groupNodesByZone + ZoneGroups / AzAwareLayout over string labels, loop for loop."""
    def group_nodes_by_zone(names):
        zones_in_order, by_zone = [], {}
        for n in names:
            z = zone_label[n]
            if z not in by_zone:
                zones_in_order.append(z)
                by_zone[z] = []
            by_zone[z].append(n)
        return zones_in_order, by_zone
    dz_order, dz = group_nodes_by_zone(drv)
    _, ez = group_nodes_by_zone(exe)
    groups = [(z, dz[z], ez[z]) for z in dz_order if z in ez]
    n_zones = len(groups)
    if kind == AZ_AWARE:
        in_zone = set()
        for _, d, e in groups:
            in_zone.update(d); in_zone.update(e)
        rest_d = [n for n in drv if n not in in_zone]
        rest_e = [n for n in exe if n not in in_zone]
        if not groups or rest_d or rest_e:
            groups.append((None, rest_d, rest_e))
    elif not groups:
        groups.append((None, [], []))          # EmptyPackingResult: one empty group, every result zone -1
    eo, do, eoff, doff = [], [], [0], [0]
    for _, d, e in groups:
        eo += e; do += d
        eoff.append(len(eo)); doff.append(len(do))
    return dict(n_zones=n_zones, n_groups=len(groups), zones=[z for z, _, _ in groups], exec_order=eo, drv_order=do,
                exec_off=eoff, drv_off=doff)


def check(drv, exe, zone, n_zone_ids, kind, label=""):
    got = device_model(drv, exe, zone, n_zone_ids, kind)
    want = literal_layout([int(x) for x in drv], [int(x) for x in exe], {i: "zone-%d" % z for i, z in enumerate(zone)}, kind)
    assert got["n_zones"] == want["n_zones"], label
    assert got["n_groups"] == want["n_groups"], label
    zog = ["zone-%d" % z if z >= 0 else None for z in got["zone_of_group"][:got["n_groups"]]]
    assert zog == want["zones"], label
    assert (got["zone_of_group"][got["n_groups"]:] == -1).all(), label
    for k in ("exec_order", "drv_order", "exec_off", "drv_off"):
        assert [int(x) for x in got[k]] == want[k], (label, k)
    for k in ("exec", "drv"):                                  # groups past the last one are empty
        assert (got[k + "_bound_off"][got["n_groups"]:] == got[k + "_off"][-1]).all(), label
    return got


def random_case(rng, n, n_zone_ids, used_zones=None):
    used = used_zones if used_zones is not None else n_zone_ids
    zone = rng.integers(0, used, n)
    if n_zone_ids > used:
        zone = rng.permutation(n_zone_ids)[:used][zone]           # unused ids anywhere in the range
    perm = rng.permutation(n)
    p_d, p_e = rng.random(), rng.random()
    drv = perm[rng.random(n) < p_d]
    exe = rng.permutation(n)[rng.random(n) < p_e]                  # a different order: interleaves the zones
    return drv, exe, zone


@pytest.mark.parametrize("kind", [SINGLE_AZ, AZ_AWARE])
def test_random_orders(kind):
    rng = np.random.default_rng(400 + kind)
    for t in range(2500):
        n = int(rng.integers(0, 60))
        Z = int(rng.integers(1, 12))
        drv, exe, zone = random_case(rng, n, Z, used_zones=int(rng.integers(1, Z + 1)))
        check(drv, exe, zone, Z, kind, f"case {t}")


@pytest.mark.parametrize("kind", [SINGLE_AZ, AZ_AWARE])
def test_label_interleaved_zones(kind):
    """A label re-sort moves nodes of a later zone ahead: the zone order follows the re-sorted driver order, not the zone
    priority of the sort."""
    rng = np.random.default_rng(7)
    for t in range(300):
        n, Z = 40, 5
        zone = np.sort(rng.integers(0, Z, n))                       # the node order sorted by zone priority ...
        label = rng.integers(-1, 3, n)
        key = np.where(label < 0, BIG, label)
        drv = np.argsort(key, kind="stable")                         # ... then re-sorted by label rank
        exe = np.argsort(np.where(rng.integers(-1, 3, n) < 0, BIG, 1), kind="stable")
        got = check(drv, exe, zone, Z, kind, f"case {t}")
        firsts = [int(np.nonzero(zone[drv] == z)[0][0]) for z in got["zone_of_group"][:got["n_zones"]]]
        assert firsts == sorted(firsts)


@pytest.mark.parametrize("kind", [SINGLE_AZ, AZ_AWARE])
def test_edges(kind):
    rng = np.random.default_rng(11)
    # driver-only and executor-only zones next to candidate zones
    zone = np.array([0, 0, 1, 1, 2, 2, 3, 3])
    drv = np.array([2, 3, 6, 4]); exe = np.array([1, 5, 7, 6])     # zone 1 driver-only, zone 0 executor-only, 3 then 2 both
    got = check(drv, exe, zone, 4, kind)
    assert got["n_zones"] == 2 and list(got["zone_of_group"][:2]) == [3, 2]
    # no candidate zone
    got = check(np.array([0, 1]), np.array([2, 3]), np.array([0, 0, 1, 1]), 2, kind)
    assert got["n_zones"] == 0 and got["n_groups"] == 1
    assert (len(got["exec_order"]), len(got["drv_order"])) == ((2, 2) if kind == AZ_AWARE else (0, 0))
    # empty orders
    got = check(np.array([], np.int64), np.array([], np.int64), np.zeros(3, np.int64), 1, kind)
    assert got["n_groups"] == 1 and got["n_zones"] == 0
    # one zone (zone_id NULL)
    drv, exe, zone = random_case(rng, 50, 1)
    got = check(drv, exe, zone, 1, kind)
    assert got["n_zones"] == (1 if len(drv) and len(exe) else 0)
    # one node per zone, and 70 zones
    for n in (1, 2, 17, 300):
        zone = rng.permutation(n)
        drv = rng.permutation(n); exe = rng.permutation(n)[: n // 2 + 1]
        check(drv, exe, zone, n, kind, f"one node per zone, n={n}")
    drv, exe, zone = random_case(rng, 3000, 70)
    got = check(drv, exe, zone, 70, kind)
    assert got["n_zones"] == 70
    # unused zone ids (only 3 of 1000 used)
    drv, exe, zone = random_case(rng, 200, 1000, used_zones=3)
    check(drv, exe, zone, 1000, kind)


def test_gp_zone_layout_struct_matches_header():
    import k8s_spark_scheduler_b200 as g
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gangpack.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %d %d\n", sizeof(gp_zone_layout), offsetof(gp_zone_layout, kind),
             offsetof(gp_zone_layout, n_zones), offsetof(gp_zone_layout, n_groups), offsetof(gp_zone_layout, n_driver),
             offsetof(gp_zone_layout, n_executor), offsetof(gp_zone_layout, reserved), offsetof(gp_zone_layout, zone_of_group),
             offsetof(gp_zone_layout, exec_off), offsetof(gp_zone_layout, exec_order), offsetof(gp_zone_layout, drv_off),
             offsetof(gp_zone_layout, drv_order), (int)GP_LAYOUT_SINGLE_AZ, (int)GP_LAYOUT_AZ_AWARE);
      return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    L = g.native.gp_zone_layout
    assert got == [ctypes.sizeof(L)] + [getattr(L, f).offset for f in ("kind", "n_zones", "n_groups", "n_driver", "n_executor", "reserved",
                                                                       "zone_of_group", "exec_off", "exec_order", "drv_off", "drv_order")] + \
        [g.native.LAYOUT_SINGLE_AZ, g.native.LAYOUT_AZ_AWARE]


def test_entry_exported_bound_and_documented():
    import k8s_spark_scheduler_b200 as g
    g.native.build()
    assert "gp_prepare_cluster_zones" in g.native.EXPORTS
    out = subprocess.check_output(["nm", "-D", "--defined-only", g.native.LIB_PATH], text=True)
    assert any(line.split()[-1] == "gp_prepare_cluster_zones" for line in out.splitlines() if " T " in line)
    assert g.native.load().gp_prepare_cluster_zones.argtypes[-1]._type_ is g.native.gp_zone_layout
    sass = subprocess.check_output(["cuobjdump", "-sass", g.native.LIB_PATH], text=True)
    for k in ("gp_zone_mark", "gp_zone_candidates", "gp_group_rank", "gp_group_offsets"):
        assert k in sass, k
        assert k in open(os.path.join(ROOT, "DESIGN.md")).read(), k
