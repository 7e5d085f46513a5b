"""CPU checks of the failover reconciler's closed form (DESIGN §2.3) against two literal restatements of
availableResourcesPerInstanceGroup + findNodes + the charge loop (EXT/failover.go:43-82, 286-436), and of the new ABI structs'
layout against a C compiler."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import reconcile_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _agree(case):
    lp, lo, loff, lav = R.literal_flat(case)
    cp, co, coff, cav, cbad = R.c_literal(case)
    fp, fo, foff, fav, fbad = R.closed_form(case)
    assert np.array_equal(lp, cp) and np.array_equal(lp, fp)
    for i in range(len(lp)):
        s = slice(loff[i], loff[i] + max(int(lp[i]), 0))
        assert np.array_equal(lo[s], co[s]) and np.array_equal(lo[s], fo[s]), i
    for d in range(3):
        assert [int(x) for x in lav[d]] == [int(x) for x in cav[d]] == [int(x) for x in fav[d]], d
    assert not cbad and not fbad
    return lp


def test_literals_and_closed_form_agree_on_random_cases():
    rng = np.random.default_rng(20261016)
    seen = {"missing": 0, "k0": 0, "partial": 0, "complete": 0, "missing_k0": 0}
    for _ in range(3000):
        case = R.random_case(rng, int(rng.integers(0, 40)), int(rng.integers(1, 6)), int(rng.integers(0, 14)), int(rng.integers(0, 60)))
        placed = _agree(case)
        _, _, count, _ = R.to_device_args(case)
        seen["missing"] += int((placed == -1).sum())
        seen["missing_k0"] += int(((placed == -1) & (count == 0)).sum())
        seen["k0"] += int(((placed == 0) & (count == 0)).sum())
        seen["partial"] += int(((placed >= 0) & (placed < count)).sum())
        seen["complete"] += int(((placed == count) & (count > 0)).sum())
    assert min(seen.values()) > 50, seen


def _one_group(alloc_cpu, exe_cpu, counts, creation=None, ready=None):
    n, q = len(alloc_cpu), len(counts)
    return dict(names=[f"n{i}" for i in range(n)], alloc=(np.array(alloc_cpu, np.int64), np.full(n, 1 << 40, np.int64), np.zeros(n, np.int64)),
                label=["a"] * n, unschedulable=None, ready=ready,
                creation=np.array(creation if creation is not None else list(range(n, 0, -1)), np.int64), overhead=None,
                res_node=np.zeros(0, np.int32), res=(np.zeros(0, np.int64),) * 3, dgroup=["a"] * q,
                exe=(np.array(exe_cpu, np.int64), np.zeros(q, np.int64), np.zeros(q, np.int64)), min=np.array(counts), running=np.zeros(q))


def test_overshoot_charge_and_exact_completion():
    # node 0 holds 2, node 1 holds 3: a driver of 4 takes 2 + 2 and charges node 0 three executors (the failed addition stays
    # in `reserved`), node 1 two; a driver of 5 completes exactly at node 1's capacity and charges it no more than it took
    case = _one_group([2000, 3000, 4000], [1000], [4])
    assert list(_agree(case)) == [4]
    assert [int(x) for x in R.literal_flat(case)[3][0]] == [-1000, 1000, 4000]
    case = _one_group([2000, 3000, 4000], [1000], [5])
    _agree(case)
    assert [int(x) for x in R.literal_flat(case)[3][0]] == [-1000, 0, 4000]


def test_incomplete_driver_charges_every_node_of_its_group():
    case = _one_group([0, 1500, -700], [1000, 1000], [10, 1])
    placed = _agree(case)
    assert list(placed) == [1, 0]
    # first driver: 1 + 2 + 1 executors charged, second: every node once more
    assert [int(x) for x in R.literal_flat(case)[3][0]] == [-2000, -1500, -2700]


def test_creation_ties_keep_node_table_order():
    case = _one_group([1000] * 4, [1000], [4], creation=[5, 7, 7, 5])
    _, out, _, _ = R.literal_flat(case)
    assert list(out) == [1, 2, 0, 3]
    _agree(case)


def test_domain_exit_is_reported_by_both_exact_restatements():
    big = (1 << 60) + 12345
    case = _one_group([1 << 60], [big, big, big], [1, 1, 1])
    _, _, _, _, cbad = R.c_literal(case)
    fbad = R.closed_form(case)[4]
    assert cbad and fbad


def test_struct_layout_matches_header():
    from k8s_spark_scheduler_b200 import native
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gangpack.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(gp_reconcile_nodes), offsetof(gp_reconcile_nodes, node_group),
             offsetof(gp_reconcile_nodes, creation), offsetof(gp_reconcile_nodes, unschedulable), offsetof(gp_reconcile_nodes, ready),
             sizeof(gp_reconcile_results), offsetof(gp_reconcile_results, executor_nodes_cap), offsetof(gp_reconcile_results, avail_cpu_milli),
             offsetof(gp_reconcile_results, avail_mem_bytes), offsetof(gp_reconcile_results, avail_gpu));
      return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "l.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "l")
        subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", exe, c])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    N, Rz = native.gp_reconcile_nodes, native.gp_reconcile_results
    want = [C.sizeof(N), N.node_group.offset, N.creation.offset, N.unschedulable.offset, N.ready.offset,
            C.sizeof(Rz), Rz.executor_nodes_cap.offset, Rz.avail_cpu_milli.offset, Rz.avail_mem_bytes.offset, Rz.avail_gpu.offset]
    assert got == want

