"""Time the driver Predicate's front end from the resident tables (gp_reservation_table_update + gp_overhead_table_update +
gp_prepare_cluster_groups_resident with overhead from the overhead table) against the per-call form
(gp_overhead_table_query + gp_prepare_cluster_groups with every reservation row).

    python tools/resident_prepare_bench.py [--reps 10] [--warmup 2] [--out FILE]

Clusters: 10 000 nodes x 100 000 reservation rows and 50 000 x 1 000 000, in ResourceReservations of 21 rows (a driver and
20 executors) on random nodes, each with the overhead records of overhead.synthetic_cluster (300 000 and 1 000 000 pods, as
in tools/overhead_table_bench.py) in a resident overhead table.  Four instance groups, three zones.  Then simulated
Predicates for a churn of 0.1 % and of 1 % of the reservation rows (whole ResourceReservations rewritten onto other nodes)
and of the pod records (deleted and re-added on another node), plus one new ResourceReservation of 21 rows and one of 20 pods
in the overhead table.  Per Predicate, in the same run, the two forms after the same overhead-table update, in alternating
order:
  resident   gp_reservation_table_update with the Predicate's delta, then gp_prepare_cluster_groups_resident with
             overhead_node_id (GetOverhead never leaves the device)
  per-call   gp_overhead_table_query over every node, then gp_prepare_cluster_groups with every row (reservations.to_usage_rows
             of the numpy mirror), from ordinary (pageable) numpy arrays and from page-locked ones (GangPacker.pinned)
Both forms read back the orders; every timed Predicate checks the resident orders, counts and get_snapshot equal to the
per-call ones.  Wall clock around each call (each ends in a stream synchronise).  The deltas and row arrays are built before
the timed loop and not timed.  Medians over --reps Predicates after --warmup, with the 10th and 90th percentiles.  Prints the
card's name and power limit, read in the same run.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import overhead as oh  # noqa: E402
from k8s_spark_scheduler_b200 import reservations as rv  # noqa: E402

GIB = 1 << 30
ROWS_PER_RR = 21


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def clock(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def stats(ts):
    return {"median": round(float(np.median(ts)), 4), "p10": round(float(np.percentile(ts, 10)), 4),
            "p90": round(float(np.percentile(ts, 90)), 4)}


def rr_rows(rng, nodes, tag):
    return {f"e{j}": (nodes[rng.integers(len(nodes))], int(rng.integers(1, 9)) * 500, int(rng.integers(1, 17)) << 28,
                      int(rng.integers(0, 8) == 0)) for j in range(ROWS_PER_RR)}


def churn(rt, ot, pods, nodes, rng, frac, tag):
    """one Predicate's worth of events -> (reservation delta, overhead delta)"""
    keys = list(rt.rrs)
    for k in rng.choice(len(keys), max(1, int(len(keys) * frac)), replace=False):
        rt.rr_set(keys[k], {n: (nodes[rng.integers(len(nodes))],) + r[1:] for n, r in rt.rrs[keys[k]].items()})
    rt.rr_set(("bench", f"new-{tag}"), rr_rows(rng, nodes, tag))
    for i in rng.choice(len(pods), max(1, int(len(pods) * frac)), replace=False):
        p = pods[i]
        ot.delete(p)
        q = dict(p, uid=f"{p['uid']}-{tag}", nodeName=nodes[rng.integers(len(nodes))])
        ot.add(q)
        pods[i] = q
    ot.rr_set((f"ns-{tag % 16}", f"bench-{tag}"), [f"bench-{tag}-exec-{e}" for e in range(20)])
    return rt.delta(), ot.delta()


def same(a, b):
    (ga, sa), (gb, sb) = a, b
    return ga.keys() == gb.keys() and all(np.array_equal(ga[k], gb[k]) for k in ga) and all(np.array_equal(x, y) for x, y in zip(sa, sb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    p = g.GangPacker()
    rows = []
    try:
        for seed, (n, n_rows, n_pods, big) in enumerate([(10_000, 100_000, 300_000, 20), (50_000, 1_000_000, 1_000_000, 40)]):
            rng = np.random.default_rng(seed)
            nodes, _, lister, rrs, soft, pods = oh.synthetic_cluster(seed, n, n_pods, big_apps=big, big_executors=2000)
            ot = oh.OverheadTable(n_slots=n_pods, n_node_ids=n, n_app_keys=1 << 16, n_app_ids=1 << 16, n_names=1 << 21)
            for pod in pods:
                ot.add(pod)
            for pod in lister.values():
                ot.lister_set(pod)
            for k, v in rrs.items():
                ot.rr_set(k, v)
            for k, v in soft.items():
                ot.soft_set(k, v)
            od = ot.delta()
            p.overhead_table_reset(**od["reset"])
            p.overhead_table_update(od)
            rt = rv.ReservationTable(n_slots=2 * n_rows, n_node_ids=n)
            mirror = rv.ReservationMirror()
            for r in range(n_rows // ROWS_PER_RR):
                rt.rr_set(("bench", f"app-{r}"), rr_rows(rng, nodes, r))
            d = rt.delta()
            mirror.apply(d)
            p.reservation_table_reset(**d["reset"])
            t_load, _ = clock(lambda: p.reservation_table_update(d))
            alloc = [rng.integers(8, 65, n) * 1000, rng.integers(32, 513, n) * GIB, rng.integers(0, 9, n)]
            ig = rng.integers(0, 4, n).astype(np.int32)
            sort = dict(zone_id=rng.integers(0, 3, n).astype(np.int32), n_zones=3, name_rank=rng.permutation(n).astype(np.int32))
            oids, ids = ot.node_ids(nodes), rt.node_ids(nodes)
            assert (oids >= 0).all()
            cap = 2 * n_rows
            pin = [p.pinned(cap, np.int32)] + [p.pinned(cap, np.int64) for _ in range(3)]
            for frac in (0.001, 0.01):
                steps = []
                for s in range(args.warmup + args.reps):
                    rd, odl = churn(rt, ot, pods, nodes, rng, frac, int(frac * 1e4) * 1000 + s)
                    mirror.apply(rd)
                    ids = rt.node_ids(nodes)
                    rnode, res = rv.to_usage_rows(mirror, ids)
                    steps.append((rd, odl, ids, rnode, res))
                t = {k: [] for k in ("overhead_update", "reservation_update", "prepare_resident", "resident_predicate", "overhead_query",
                                     "prepare_per_call_pageable", "per_call_predicate_pageable", "prepare_per_call_pinned",
                                     "per_call_predicate_pinned")}
                for s, (rd, odl, ids, rnode, res) in enumerate(steps):
                    t_ou, _ = clock(lambda: p.overhead_table_update(odl))

                    def resident():
                        t_ru, _ = clock(lambda: p.reservation_table_update(rd))
                        t_pr, got = clock(lambda: p.prepare_cluster_groups_resident(ids, alloc, None, ig, 4, overhead_node_id=oids, **sort))
                        return (t_ru, t_pr), (got, p.get_snapshot())

                    def per_call(rows_in):
                        t_q, q = clock(lambda: p.overhead_table_query(oids, has_reservation=False))
                        t_pc, got = clock(lambda: p.prepare_cluster_groups(alloc, q[0], rows_in[0], rows_in[1:], ig, 4, **sort))
                        return (t_q, t_pc), (got, p.get_snapshot())

                    k = len(rnode)
                    pinned_rows = [pin[0][:k], pin[1][:k], pin[2][:k], pin[3][:k]]
                    for dst, src in zip(pinned_rows, (rnode,) + tuple(res)):
                        dst[...] = src
                    if s % 2:
                        r_t, r_out = resident()
                        pg_t, pg_out = per_call((rnode,) + tuple(res))
                    else:
                        pg_t, pg_out = per_call((rnode,) + tuple(res))
                        r_t, r_out = resident()
                    pn_t, pn_out = per_call(pinned_rows)
                    assert same(r_out, pg_out) and same(r_out, pn_out), "resident and per-call Predicates disagree"
                    if s >= args.warmup:
                        vals = (t_ou, r_t[0], r_t[1], t_ou + r_t[0] + r_t[1], pg_t[0], pg_t[1], t_ou + pg_t[0] + pg_t[1], pn_t[1],
                                t_ou + pn_t[0] + pn_t[1])
                        for key, v in zip(t, vals):
                            t[key].append(v)
                row = dict(nodes=n, reservation_rows=len(steps[-1][3]), pod_records=n_pods, churn_fraction=frac,
                           reservation_slot_writes_per_update=int(np.median([len(st[0]["slot"]) for st in steps])),
                           initial_load_update_ms=round(t_load, 3), ms={key: stats(v) for key, v in t.items()},
                           resident_h2d_bytes=8 * n + 8 * 3 * n, per_call_h2d_bytes=28 * len(steps[-1][3]) + 48 * n + 4 * n,
                           per_call_query_d2h_bytes=48 * n, parity_checked_predicates=len(steps))
                rows.append(row)
                print(json.dumps(row), flush=True)
    finally:
        p.close()
    res = {"card": card(), "rows": rows}
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
