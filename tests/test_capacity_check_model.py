"""CPU: the criterion gp_exceeds_cluster_capacity evaluates (DESIGN §2.2) against DoesPodExceedClusterCapacity itself.

Every case packs each driver literally through oracle/pyref.py -- zero-usage metadata, the affinity nodes in three random
lister orders, each of the five packers -- and requires the three answers to agree with each other and with the restated
criterion (T + M >= k, per zone and with the positivity rule for the single-AZ packers).
"""
import ctypes
import os
import random
import subprocess
import tempfile

import pytest

import capacity_ref as cr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GI = 1 << 30


def _node(rng):
    kind = rng.random()
    if kind < 0.1:
        return (rng.choice([0, 1000]), rng.choice([0, GI]), 0), (0, 0, 0)          # zero dimensions
    gpu = rng.choice([0, 0, 1, 2, 8])
    alloc = (rng.choice([2000, 4000, 8000, 16000, 7500]), rng.choice([4, 8, 16, 32]) * GI, gpu)
    over = (0, 0, 0)
    r = rng.random()
    if r < 0.3:
        over = (rng.choice([0, 500, 1000]), rng.choice([0, GI // 2, GI]), 0)
    elif r < 0.4:                                                                  # negative schedulable dimensions
        over = (alloc[0] + rng.choice([1, 1000]), rng.choice([0, alloc[1] + 1]), rng.choice([0, gpu + 1]))
    return alloc, over


def _shape(rng, zero_p):
    if rng.random() < zero_p:
        return (0, 0, 0)
    return (rng.choice([0, 1, 500, 1000, 2000, 3000]), rng.choice([0, 1, GI // 4, GI, 2 * GI, 3 * GI]), rng.choice([0, 0, 0, 1, 2]))


def _case(rng):
    n = rng.randint(1, 7)
    n_zones = rng.randint(1, 3)
    n_groups = rng.randint(1, 3)
    names = [f"node-{i}" for i in range(n)]
    alloc, over, zones, group = {}, {}, {}, {}
    for nm in names:
        alloc[nm], over[nm] = _node(rng)
        zones[nm] = f"zone-{rng.randrange(n_zones)}" if rng.random() < 0.9 else "default"
        group[nm] = rng.randrange(-1, n_groups)
    drivers = []
    for _ in range(rng.randint(1, 3)):
        drv, exe = _shape(rng, 0.15), _shape(rng, 0.15)
        cls = rng.randrange(-1, n_groups + 1)                                      # n_groups: an empty or absent class
        members = [nm for nm in names if cls == -1 or group[nm] == cls]
        sched = [(zones[nm], cr.pyref.sub(alloc[nm], over[nm])) for nm in members]
        if exe == (0, 0, 0):
            ks = [0, 1, rng.randint(2, 40)]                                          # unlimited capacity: small counts
        else:
            b = cr.boundary_k(sched, drv, exe)
            ks = [0, rng.randint(0, 12)]
            if b is not None and b <= 200:
                ks += [b, b + 1] + ([b - 1] if b >= 1 else [])
        for k in ks:
            drivers.append((drv, exe, k, members, sched))
    return alloc, over, zones, drivers


def test_criterion_matches_literal_marker():
    rng = random.Random(20261015)
    checked = flipped = 0
    for case in range(2500):
        alloc, over, zones, drivers = _case(rng)
        for drv, exe, k, members, sched in drivers:
            for packer in cr.PACKERS:
                want = cr.model_exceeds(packer, sched, drv, exe, k)
                answers = set()
                for _ in range(3):
                    order = list(members)
                    rng.shuffle(order)
                    answers.add(cr.literal_exceeds(packer, alloc, over, zones, order, drv, exe, k))
                assert len(answers) == 1, (case, packer, drv, exe, k)
                assert answers.pop() == want, (case, packer, drv, exe, k, sched)
                checked += 1
                flipped += want
    assert checked > 20000 and 0.1 < flipped / checked < 0.9


@pytest.mark.parametrize("packer", cr.PACKERS)
def test_boundary_at_t_plus_m(packer):
    # two 8-core nodes, 4 executors each, driver takes one executor's room on its node: T + M = 8 - 1 = 7
    alloc = {"a": (8000, 8 * GI, 0), "b": (8000, 8 * GI, 0)}
    zones = {"a": "z", "b": "z"}
    sched = [("z", alloc["a"]), ("z", alloc["b"])]
    drv, exe = (1000, GI, 0), (2000, 2 * GI, 0)
    assert cr.boundary_k(sched, drv, exe) == 7
    for k, exceeds in ((7, False), (8, True)):
        assert cr.model_exceeds(packer, sched, drv, exe, k) is exceeds
        assert cr.literal_exceeds(packer, alloc, {}, zones, ["b", "a"], drv, exe, k) is exceeds


def test_minimal_fragmentation_all_zero_executor():
    # every capacity is Go's max int: (executorCount + maxCapacity) / 2 wraps negative and the first search comes back empty;
    # the full search then succeeds whenever some node fits -- what T + M >= k says
    alloc = {"a": (4000, 4 * GI, 0), "b": (1000, GI, 0)}
    zones = {"a": "z1", "b": "z2"}
    for drv, k in (((0, 0, 0), 5), ((1000, GI, 0), 3), ((4000, 4 * GI, 0), 1), ((5000, GI, 0), 1), ((1000, GI, 0), 0)):
        sched = [(zones[n], alloc[n]) for n in alloc]
        for packer in cr.PACKERS:
            want = cr.model_exceeds(packer, sched, drv, (0, 0, 0), k)
            assert cr.literal_exceeds(packer, alloc, {}, zones, ["a", "b"], drv, (0, 0, 0), k) is want, (packer, drv, k)


def test_single_az_positivity_rule():
    alloc = {"a": (4000, 4 * GI, 0)}
    zones = {"a": "z"}
    sched = [("z", alloc["a"])]
    # all-zero driver: single-az-tightly-pack needs an executor with a positive request, minimal fragmentation never counts it
    for exe, k, tp, mf in (((1000, 0, 0), 1, False, True), ((1000, 0, 0), 0, True, True), ((0, 0, 0), 3, True, True)):
        assert cr.model_exceeds("single-az-tightly-pack", sched, (0, 0, 0), exe, k) is tp
        assert cr.model_exceeds("single-az-minimal-fragmentation", sched, (0, 0, 0), exe, k) is mf
        assert cr.literal_exceeds("single-az-tightly-pack", alloc, {}, zones, ["a"], (0, 0, 0), exe, k) is tp
        assert cr.literal_exceeds("single-az-minimal-fragmentation", alloc, {}, zones, ["a"], (0, 0, 0), exe, k) is mf
        assert cr.model_exceeds("tightly-pack", sched, (0, 0, 0), exe, k) is False


def test_capacity_nodes_struct_layout_matches_header():
    import k8s_spark_scheduler_b200 as g
    native = g.native
    fields = [f[0] for f in native.gp_capacity_nodes._fields_]
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "gangpack.h"\nint main(void) {\n  printf("%zu", sizeof(gp_capacity_nodes));\n'
           + "".join(f'  printf(" %zu", offsetof(gp_capacity_nodes, {f}));\n' for f in fields)
           + '  printf(" %d %d %d %d %d\\n", GP_BP_TIGHTLY_PACK, GP_BP_DISTRIBUTE_EVENLY, GP_BP_AZ_AWARE_TIGHTLY_PACK,\n'
             '         GP_BP_SINGLE_AZ_TIGHTLY_PACK, GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION);\n  return 0; }\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    S = native.gp_capacity_nodes
    assert got[:1 + len(fields)] == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in fields]
    assert got[1 + len(fields):] == [native.BINPACKERS[p] for p in cr.PACKERS] == [0, 1, 2, 3, 4]
    assert "gp_exceeds_cluster_capacity" in native.EXPORTS
