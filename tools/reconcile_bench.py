"""Time gp_reconcile_find_nodes -- the failover reconciler's node choice for every stale driver in one device call -- against the
string-keyed C literal of the same loop (tests/reconcile_oracle.c, restated, not Go), run single-threaded on the host.

    python tools/reconcile_bench.py [--reps 10] [--warmup 2] [--out FILE]

Sizes: 10 000 nodes / 16 instance groups / 1 000 stale drivers and 50 000 / 64 / 10 000, each with 100 000 reservation rows
(hard and soft alike, some on nodes outside the table), creation ties, unschedulable and not-ready nodes, and 1 % of the drivers
asking for more than their group holds.  Wall clock (time.perf_counter) around each complete call: the device call ends in a
stream synchronise; both sides have their inputs marshalled beforehand except what each call itself copies.  The two sides
alternate, median and best of --reps repetitions after --warmup.  Outputs (placed, every ExecutorNodes slice, the availability
after the loop) are checked equal.  Prints the card's name and power limit with the numbers.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import k8s_spark_scheduler_b200 as g  # noqa: E402
import reconcile_ref as R  # noqa: E402

SIZES = [(10_000, 16, 1_000), (50_000, 64, 10_000)]
ROWS = 100_000


def make_case(seed, n, groups, q):
    rng = np.random.default_rng(seed)
    case = R.random_case(rng, n, groups, q, ROWS)
    case["alloc"] = (case["alloc"][0] * 4, case["alloc"][1] * 4, case["alloc"][2])
    case["min"] = np.where(rng.random(q) < 0.01, 50_000, case["min"])
    return case


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    p = g.GangPacker(device=0)
    print("card:", card())
    rows = []
    try:
        for n, groups, q in SIZES:
            case = make_case(n + q, n, groups, q)
            dev = _device(p, case)
            lit = R.c_literal_bound(case)
            d, c = dev(), lit()
            assert np.array_equal(d[0], c[0]) and np.array_equal(d[2], c[2])
            for i in np.nonzero(c[0] > 0)[0]:
                assert np.array_equal(d[1][c[2][i]:c[2][i] + c[0][i]], c[1][c[2][i]:c[2][i] + c[0][i]])
            assert all(np.array_equal(x, y) for x, y in zip(d[3], c[3])) and not c[4]
            for _ in range(args.warmup):
                dev(); lit()
            td, tc = [], []
            for _ in range(args.reps):
                t = time.perf_counter(); dev(); td.append(time.perf_counter() - t)
                t = time.perf_counter(); lit(); tc.append(time.perf_counter() - t)
            row = dict(nodes=n, groups=groups, drivers=q, rows=ROWS, placed=int(np.maximum(d[0], 0).sum()),
                       device_ms_median=1e3 * float(np.median(td)), device_ms_best=1e3 * min(td),
                       c_literal_ms_median=1e3 * float(np.median(tc)), c_literal_ms_best=1e3 * min(tc), outputs_equal=True)
            print(json.dumps(row))
            rows.append(row)
    finally:
        p.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), baseline="C literal, single-threaded, restated, not Go", results=rows), f, indent=1)


def _device(p, case):
    """The call's arguments converted to their ABI dtypes once -> a zero-argument callable (the binding's struct marshalling and
    the call itself, which ends in a stream synchronise)."""
    ng, dg, count, G = R.to_device_args(case)
    i64 = lambda t: tuple(None if x is None else np.ascontiguousarray(x, np.int64) for x in t)
    alloc, over, res, exe = i64(case["alloc"]), i64(case["overhead"]), i64(case["res"]), i64(case["exe"])
    rn, cr = np.ascontiguousarray(case["res_node"], np.int32), np.ascontiguousarray(case["creation"], np.int64)
    fu, fr = np.ascontiguousarray(case["unschedulable"], np.uint8), np.ascontiguousarray(case["ready"], np.uint8)
    apps = dict(exe_cpu=exe[0], exe_mem=exe[1], exe_gpu=exe[2], count=count, group=dg)
    return lambda: p.reconcile_find_nodes(alloc, over, rn, res, ng, cr, apps, G, unschedulable=fu, ready=fr)


if __name__ == "__main__":
    main()
