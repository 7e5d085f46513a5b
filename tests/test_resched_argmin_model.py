"""CPU model of gp_reschedule_from_reservations (no GPU): the arg-min formulation of DESIGN.md §2 -- first fit = the smallest
key (L, P, mem, cpu, name) among the candidates the executor fits on, minimal fragmentation = the smallest (not hosting,
capacity, key) among the candidates with capacity >= 1 -- equals the decision over the sorted PotentialNodes order of the
literal rescheduleExecutor chain (tests/reschedule_ref.py over oracle/pyref.py), and its ambiguity flag equals a brute force
over every order the reference's unstable sort may produce.  Also: the literal filterNodesToZone /
getCommonZoneForExecutorsApplication error cases, and the gp_reschedule_scope layout against a C compiler."""
import ctypes
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import reschedule_ref as rr
from reschedule_ref import ZONE_LABEL, ReferenceError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_case(rng):
    tie = rng.random() < 0.4                                     # tie mode: two (mem, cpu) levels, gpu free to differ
    n = int(rng.integers(0, 7 if tie else 10))                   # runs stay short enough for the brute force below
    names = ["n%02d" % int(x) for x in rng.permutation(40)[:n]]
    nz = int(rng.integers(1, 4))
    zl = ["zone-%d" % int(z) for z in rng.integers(0, nz, n)]
    scoped = n > 0 and rng.random() < 0.4
    missing = (rng.random(n) < 0.15) & (not scoped)            # a missing label is only legal without a scope
    labels = {nm: ({} if missing[i] else {ZONE_LABEL: zl[i]}) for i, nm in enumerate(names)}
    # the sorter's zone is the BETA label ("default" when absent, LIB/resources/resources.go:78-81), not the topology label
    # filterNodesToZone reads (SURVEY App. B5): absent, the same zone, or another one
    beta = [[None, zl[i], "zone-%d" % int(rng.integers(0, nz + 1))][int(rng.integers(0, 3))] for i in range(n)]
    sort_zone = {nm: beta[i] if beta[i] is not None else "default" for i, nm in enumerate(names)}
    small = rng.random() < 0.5                                   # small ranges: equal (mem, cpu) with differing gpu, equal totals
    lo, hi = (2, 4) if small else (0, 9)
    alloc = {nm: (int(rng.integers(lo, hi)) * 1000, int(rng.integers(lo, hi)) * 1024, int(rng.integers(0, 3))) for nm in names}
    over = {nm: (int(rng.integers(0, 2)) * 500, int(rng.integers(0, 2)) * 512, int(rng.integers(0, 2) * (rng.random() < 0.3)))
            for nm in names}
    R = int(rng.integers(0, 5 if small else 12))
    res_nodes = [names[int(rng.integers(0, n))] if n and rng.random() < 0.9 else "gone" for _ in range(R)]
    reservations = [(nd, (int(rng.integers(0, 3)) * 500, int(rng.integers(0, 3)) * 512, int(rng.integers(0, 2)))) for nd in res_nodes]
    if tie:
        alloc = {nm: (v * 1000, v * 1024, int(rng.integers(0, 3))) for nm, v in zip(names, rng.integers(2, 4, n).tolist())}
        over = {nm: (0, 0, int(o)) for nm, o in zip(names, rng.integers(0, 2, n).tolist())}
        reservations = [(nd, (0, 0, g)) for nd, (_, _, g) in reservations]
        if rng.random() < 0.6:                                   # no beta label anywhere: one sorter zone, "default"
            sort_zone = {nm: "default" for nm in names}
    unsched = {nm for nm in names if rng.random() < 0.15}
    not_ready = {nm for nm in names if rng.random() < 0.1}
    lab = None
    if rng.random() < 0.5:
        lab = {nm: int(rng.integers(-1, 3)) for nm in names}
    exe = tuple(int(rng.integers(0, 3 if d < 2 else 2)) * m for d, m in enumerate((500, 512, 1))) if rng.random() < 0.9 else (0, 0, 0)
    min_frag = bool(rng.random() < 0.5)
    hosting = {nm for nm in names if rng.random() < 0.3}
    common = None
    if scoped:
        common = "zone-%d" % int(rng.integers(0, nz + 1))       # zone-nz: no node kept
    return dict(names=names, labels=labels, sort_zone=sort_zone, alloc=alloc, over=over, reservations=reservations,
                unsched=unsched, not_ready=not_ready, lab=lab, exe=exe, min_frag=min_frag, hosting=hosting, common=common)


def model(c):
    """The device algorithm over node-table indices: per-node values, member and candidate masks, one arg-min."""
    names = c["names"]
    n = len(names)
    idx = {nm: i for i, nm in enumerate(names)}
    al = c["alloc"]
    meta, _ = rr.pyref.node_scheduling_metadata(al, c["over"], c["reservations"])
    ff = rr.first_fit_available(al, c["over"], c["reservations"])
    interned = {}
    zone = [interned.setdefault(c["sort_zone"][nm], len(interned)) for nm in names]
    rank = {nm: r for r, nm in enumerate(sorted(names))}
    member = [c["common"] is None or c["labels"][nm].get(ZONE_LABEL) == c["common"] for nm in names]
    cand = [member[i] and nm not in c["unsched"] and nm not in c["not_ready"] for i, nm in enumerate(names)]
    lab = None if c["lab"] is None else [c["lab"][nm] for nm in names]
    w, amb = rr.decide([meta[nm] for nm in names], [ff[nm] for nm in names], [c["over"][nm] for nm in names], zone,
                       [rank[nm] for nm in names], member, cand, lab, c["exe"], c["min_frag"], {idx[h] for h in c["hosting"]})
    return (names[w] if w >= 0 else None), amb


def literal(c):
    lab = None if c["lab"] is None else {nm: r for nm, r in c["lab"].items() if r >= 0}
    order, meta, ff, ov = rr.executor_state(c["names"], c["labels"], c["sort_zone"], c["alloc"], c["over"], c["reservations"],
                                            c["unsched"], c["not_ready"], lab, c["common"])
    got = rr.choose(c["exe"], c["min_frag"], c["hosting"], order, meta, ff, ov)
    # every order the unstable sort may produce: same label key, zone priority, memory, cpu; differing gpu unordered
    labkey = (lambda nm: 0) if lab is None else (lambda nm: lab.get(nm, 1 << 31))
    prio = _zone_prio(meta, c["sort_zone"])
    key_of = lambda nm: (labkey(nm), prio[c["sort_zone"][nm]], meta[nm][1], meta[nm][0])
    alt = {rr.choose(c["exe"], c["min_frag"], c["hosting"], o, meta, ff, ov)
           for o in rr.tie_permutations(order, key_of, lambda nm: meta[nm][2], lambda nm: nm, limit=8)}
    return got, any(a != got for a in alt)


def zone_tie_choices(c):
    """Equal zone totals are ordered by the reference's unstable sort.Slice too (nodesorting.go:102-104, SURVEY App. B6); the
    device orders them by zone id.  -> None when the kept zones' (mem, cpu) totals are distinct, else every decision the
    literal chain takes over some order of the zones (node lists regrouped zone by zone: the first-seen order decides)."""
    lab = None if c["lab"] is None else {nm: r for nm, r in c["lab"].items() if r >= 0}
    order, meta, ff, ov = rr.executor_state(c["names"], c["labels"], c["sort_zone"], c["alloc"], c["over"], c["reservations"],
                                            c["unsched"], c["not_ready"], lab, c["common"])
    tot = {}
    for nm in meta:
        m, cp = tot.get(c["sort_zone"][nm], (0, 0))
        tot[c["sort_zone"][nm]] = (m + meta[nm][1], cp + meta[nm][0])
    if len(set(tot.values())) == len(tot):
        return None
    out = set()
    for zs in itertools.permutations(tot):
        nodes = [nm for z in zs for nm in c["names"] if c["sort_zone"][nm] == z] + [nm for nm in c["names"] if nm not in meta]
        o, m2, f2, v2 = rr.executor_state(nodes, c["labels"], c["sort_zone"], c["alloc"], c["over"], c["reservations"],
                                          c["unsched"], c["not_ready"], lab, c["common"])
        out.add(rr.choose(c["exe"], c["min_frag"], c["hosting"], o, m2, f2, v2))
    return out


def _zone_prio(meta, sort_zone):
    tot, first = {}, {}
    for nm in meta:
        z = sort_zone[nm]
        first.setdefault(z, len(first))
        m, cp = tot.get(z, (0, 0))
        tot[z] = (m + meta[nm][1], cp + meta[nm][0])
    zs = sorted(tot, key=lambda z: (tot[z][0], tot[z][1], first[z]))
    return {z: p for p, z in enumerate(zs)}


def test_argmin_equals_sorted_order_and_brute_force_ambiguity():
    rng = np.random.default_rng(20261015)
    seen = {"amb": 0, "none": 0, "scoped": 0, "ff": 0, "mf": 0, "host_win": 0, "zone_ties": 0}
    for t in range(6000):
        c = random_case(rng)
        got, got_amb = model(c)
        ties = zone_tie_choices(c)
        if ties is not None:                      # zones with equal totals: the device's id order is one admissible order
            assert got in ties, (t, c, got, ties)
            seen["zone_ties"] += 1
            continue
        want, want_amb = literal(c)
        assert got == want, (t, c, got, want)
        assert got_amb == want_amb, (t, c, got, want, got_amb, want_amb)
        seen["amb"] += got_amb
        seen["none"] += got is None
        seen["scoped"] += c["common"] is not None
        seen["mf" if c["min_frag"] else "ff"] += 1
        seen["host_win"] += c["min_frag"] and got in c["hosting"]
    assert all(v > 50 for v in seen.values()), seen


def test_empty_candidate_sets():
    rng = np.random.default_rng(7)
    c = random_case(rng)
    while len(c["names"]) < 3:
        c = random_case(rng)
    c["unsched"] = set(c["names"])                               # no executor candidate
    assert model(c)[0] is None and literal(c)[0] is None
    c["unsched"] = set()
    c["common"] = "zone-nowhere"                                 # every node filtered out
    for nm in c["names"]:
        c["labels"][nm] = {ZONE_LABEL: "zone-0"}
    assert model(c)[0] is None and literal(c)[0] is None


def test_sorter_zone_is_the_beta_label():
    """a: 8 cores / 8 GiB in topology zone z1; b, c: 6 / 6 in z2.  Without the beta label every node sorts in zone "default"
    and the reference chooses b; sorting by the topology label would choose a (z1 has the smaller totals)."""
    names = ["a", "b", "c"]
    labels = {"a": {ZONE_LABEL: "z1"}, "b": {ZONE_LABEL: "z2"}, "c": {ZONE_LABEL: "z2"}}
    alloc = {"a": (8000, 8 << 30, 0), "b": (6000, 6 << 30, 0), "c": (6000, 6 << 30, 0)}
    over = {nm: (0, 0, 0) for nm in names}
    exe = (1000, 1 << 30, 0)
    base = dict(names=names, labels=labels, alloc=alloc, over=over, reservations=[], unsched=set(), not_ready=set(), lab=None,
                exe=exe, min_frag=False, hosting=set(), common=None)
    c = dict(base, sort_zone={nm: "default" for nm in names})
    assert literal(c)[0] == "b" and model(c)[0] == "b"
    c = dict(base, sort_zone={nm: labels[nm][ZONE_LABEL] for nm in names})      # beta label = topology label
    assert literal(c)[0] == "a" and model(c)[0] == "a"
    c = dict(base, sort_zone={nm: "elsewhere" for nm in names}, common="z2")     # scope by topology, sort by beta
    assert literal(c)[0] == "b" and model(c)[0] == "b"


def test_filter_nodes_to_zone_literal():
    labels = {"a": {ZONE_LABEL: "z1"}, "b": {ZONE_LABEL: "z2"}, "c": {ZONE_LABEL: "z1"}, "d": {}}
    assert rr.filter_nodes_to_zone(["a", "b", "c"], labels, "z1") == ["a", "c"]
    assert rr.filter_nodes_to_zone(["a", "b", "c"], labels, "z3") == []
    with pytest.raises(ReferenceError, match="Could not read zone label"):
        rr.filter_nodes_to_zone(["a", "d"], labels, "z1")       # the unlabelled node is not even in the zone
    with pytest.raises(ReferenceError, match="Could not read zone label"):
        rr.filter_nodes_to_zone(["d", "a"], labels, "z2")


def test_common_zone_literal():
    nl = {"a": {ZONE_LABEL: "z1"}, "b": {ZONE_LABEL: "z2"}, "c": {ZONE_LABEL: "z1"}, "d": {}}
    ex = {"spark-app-id": "app"}
    assert rr.get_common_zone_for_executors_application(ex, [("Running", "a"), ("Running", "c"), ("Pending", "b")], nl) == ("z1", True)
    assert rr.get_common_zone_for_executors_application(ex, [("Running", "a"), ("Running", "b")], nl) == ("", False)
    with pytest.raises(ReferenceError, match="no scheduled pods"):
        rr.get_common_zone_for_executors_application(ex, [("Pending", "a")], nl)
    with pytest.raises(ReferenceError, match="Spark app id"):
        rr.get_common_zone_for_executors_application({}, [("Running", "a")], nl)
    with pytest.raises(ReferenceError, match="Could not read zone label"):
        rr.get_common_zone_for_executors_application(ex, [("Running", "d")], nl)
    with pytest.raises(ReferenceError, match="not found"):
        rr.get_common_zone_for_executors_application(ex, [("Running", "x")], nl)


def test_scope_struct_layout_matches_header():
    import k8s_spark_scheduler_b200 as g
    native = g.native
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gangpack.h"
    int main(void) {
      printf("%zu %zu %zu %zu\n", sizeof(gp_reschedule_scope), offsetof(gp_reschedule_scope, keep_topology_zone),
             offsetof(gp_reschedule_scope, reserved), offsetof(gp_reschedule_scope, topology_zone));
      return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    S = native.gp_reschedule_scope
    assert got == [ctypes.sizeof(S), S.keep_topology_zone.offset, S.reserved.offset, S.topology_zone.offset]
    assert "gp_reschedule_from_reservations" in native.EXPORTS
