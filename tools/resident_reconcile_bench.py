"""Time the failover reconciler and the unschedulable-pod marker from the resident tables against their per-call forms.

    python tools/resident_reconcile_bench.py [--reps 10] [--warmup 2] [--out FILE]

Reconcile.  The clusters of tools/resident_prepare_bench.py: 10 000 nodes x 100 000 reservation rows and 50 000 x 1 000 000
(ResourceReservations of 21 rows on random nodes), each with the overhead records of overhead.synthetic_cluster in a resident
overhead table; 16 instance groups, 200 stale drivers of 1-40 missing executors.  Simulated reconciles for a churn of 0.1 %
and 1 % of the reservation rows and of the pod records.  Per reconcile, after the same overhead-table update, in alternating
order:
  resident   gp_reservation_table_update with the reconcile's delta, then gp_reconcile_find_nodes_resident with
             overhead_node_id (neither a reservation row nor GetOverhead crosses to the host)
  per-call   gp_overhead_table_query over every node, then gp_reconcile_find_nodes with every row (reservations.to_usage_rows of
             the numpy mirror), from pageable numpy arrays and from page-locked ones (GangPacker.pinned)
Marker.  10 000 and 50 000 nodes with the same overhead tables, 1 000 stale drivers, four affinity classes, three zones,
single-az-tightly-pack: gp_exceeds_cluster_capacity_resident against gp_overhead_table_query + gp_exceeds_cluster_capacity.

Every timed pair is checked equal (placed, every ExecutorNodes slice and the availability; exceeds).  Wall clock around each
call (each ends in a stream synchronise); deltas and row arrays are built before the timed loop.  Medians over --reps after
--warmup, with the 10th and 90th percentiles.  Prints the card's name and power limit, read in the same run.  Needs a GPU."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import overhead as oh  # noqa: E402
from k8s_spark_scheduler_b200 import reservations as rv  # noqa: E402
from resident_prepare_bench import GIB, ROWS_PER_RR, card, churn, clock, rr_rows, stats  # noqa: E402

GROUPS, STALE, MARKER_STALE = 16, 200, 1000


def defined(r):
    placed, execn, off, av = r
    return placed, [execn[off[i]:off[i] + max(int(placed[i]), 0)] for i in range(len(placed))], av


def same(a, b):
    (pa, sa, aa), (pb, sb, ab) = defined(a), defined(b)
    return (np.array_equal(pa, pb) and all(np.array_equal(x, y) for x, y in zip(sa, sb)) and
            all(np.array_equal(x, y) for x, y in zip(aa, ab)))


def overhead_table(p, seed, n, n_pods, big):
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
    return nodes, pods, ot


def reconcile_rows(p, args, seed, n, n_rows, n_pods, big):
    rng = np.random.default_rng(seed)
    nodes, pods, ot = overhead_table(p, seed, n, n_pods, big)
    rt = rv.ReservationTable(n_slots=2 * n_rows, n_node_ids=n)
    mirror = rv.ReservationMirror()
    for r in range(n_rows // ROWS_PER_RR):
        rt.rr_set(("bench", f"app-{r}"), rr_rows(rng, nodes, r))
    d = rt.delta()
    mirror.apply(d)
    p.reservation_table_reset(**d["reset"])
    p.reservation_table_update(d)
    alloc = [rng.integers(8, 65, n) * 1000, rng.integers(32, 513, n) * GIB, rng.integers(0, 9, n)]
    node_group = rng.integers(0, GROUPS, n).astype(np.int32)
    creation = rng.integers(0, 1 << 40, n).astype(np.int64)
    ready = (rng.random(n) > 0.02).astype(np.uint8)
    apps = dict(exe_cpu=rng.integers(1, 9, STALE) * 500, exe_mem=rng.integers(1, 17, STALE) * (GIB // 2),
                exe_gpu=(rng.random(STALE) < 0.1).astype(np.int64), count=rng.integers(1, 41, STALE).astype(np.int32),
                group=rng.integers(0, GROUPS, STALE).astype(np.int32))
    nkw = dict(ready=ready)
    oids = ot.node_ids(nodes)
    cap = 2 * n_rows
    pin = [p.pinned(cap, np.int32)] + [p.pinned(cap, np.int64) for _ in range(3)]
    out = []
    for frac in (0.001, 0.01):
        steps = []
        for s in range(args.warmup + args.reps):
            rd, odl = churn(rt, ot, pods, nodes, rng, frac, int(frac * 1e4) * 1000 + s)
            mirror.apply(rd)
            ids = rt.node_ids(nodes)
            rnode, res = rv.to_usage_rows(mirror, ids)
            steps.append((rd, odl, ids, rnode, res))
        t = {k: [] for k in ("overhead_update", "reservation_update", "reconcile_resident", "resident_total", "overhead_query",
                             "reconcile_per_call_pageable", "per_call_total_pageable", "reconcile_per_call_pinned", "per_call_total_pinned")}
        for s, (rd, odl, ids, rnode, res) in enumerate(steps):
            t_ou, _ = clock(lambda: p.overhead_table_update(odl))

            def resident():
                t_ru, _ = clock(lambda: p.reservation_table_update(rd))
                t_rc, got = clock(lambda: p.reconcile_find_nodes_resident(ids, alloc, None, node_group, creation, apps, GROUPS,
                                                                          overhead_node_id=oids, **nkw))
                return (t_ru, t_rc), got

            def per_call(rows_in):
                t_q, q = clock(lambda: p.overhead_table_query(oids, has_reservation=False))
                t_pc, got = clock(lambda: p.reconcile_find_nodes(alloc, q[0], rows_in[0], rows_in[1:], node_group, creation, apps, GROUPS,
                                                                 **nkw))
                return (t_q, t_pc), got

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
            assert same(r_out, pg_out) and same(r_out, pn_out), "resident and per-call reconciles disagree"
            if s >= args.warmup:
                vals = (t_ou, r_t[0], r_t[1], t_ou + r_t[0] + r_t[1], pg_t[0], pg_t[1], t_ou + pg_t[0] + pg_t[1], pn_t[1],
                        t_ou + pn_t[0] + pn_t[1])
                for key, v in zip(t, vals):
                    t[key].append(v)
        placed = np.asarray(r_out[0])
        row = dict(entry="reconcile", nodes=n, reservation_rows=len(steps[-1][3]), pod_records=n_pods, churn_fraction=frac,
                   instance_groups=GROUPS, stale_drivers=STALE, drivers_placed_in_full=int((placed == apps["count"]).sum()),
                   ms={key: stats(v) for key, v in t.items()}, parity_checked=len(steps))
        out.append(row)
        print(json.dumps(row), flush=True)
    return out


def marker_row(p, args, seed, n, n_pods, big):
    rng = np.random.default_rng(100 + seed)
    nodes, _, ot = overhead_table(p, seed, n, n_pods, big)
    oids = ot.node_ids(nodes)
    alloc = [rng.integers(8, 65, n) * 1000, rng.integers(32, 513, n) * GIB, rng.integers(0, 9, n)]
    zone, group = rng.integers(0, 3, n).astype(np.int32), rng.integers(-1, 4, n).astype(np.int32)
    q = MARKER_STALE
    apps = dict(drv_cpu=rng.choice([500, 1000, 2000], q), drv_mem=rng.choice([GIB, 2 * GIB], q), drv_gpu=np.zeros(q, np.int64),
                exe_cpu=rng.choice([500, 1000, 2000, 8000], q), exe_mem=rng.choice([GIB, 4 * GIB, 16 * GIB], q),
                exe_gpu=np.zeros(q, np.int64), count=rng.integers(0, 3 * n, q).astype(np.int32), group=rng.integers(-1, 4, q).astype(np.int32))
    kw = dict(zone_id=zone, n_zones=3, node_group=group, n_groups=4)
    bp = g.native.BP_SINGLE_AZ_TIGHTLY_PACK
    t = {"resident": [], "overhead_query": [], "per_call": [], "per_call_total": []}
    for s in range(args.warmup + args.reps):
        def resident():
            return clock(lambda: p.exceeds_cluster_capacity_resident(alloc, oids, apps, bp, **kw))

        def per_call():
            t_q, qr = clock(lambda: p.overhead_table_query(oids, has_reservation=False))
            t_pc, got = clock(lambda: p.exceeds_cluster_capacity(alloc, apps, bp, overhead=qr[1], **kw))
            return (t_q, t_pc), got
        if s % 2:
            tr, a = resident()
            tp, b = per_call()
        else:
            tp, b = per_call()
            tr, a = resident()
        assert np.array_equal(a, b), "resident and per-call marker sweeps disagree"
        if s >= args.warmup:
            for key, v in zip(t, (tr, tp[0], tp[1], tp[0] + tp[1])):
                t[key].append(v)
    row = dict(entry="marker", nodes=n, pod_records=n_pods, stale_drivers=q, packer="single-az-tightly-pack",
               exceeding=int(a.sum()), ms={key: stats(v) for key, v in t.items()}, parity_checked=args.warmup + args.reps)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    c = card()
    print(json.dumps({"card": c}), flush=True)
    p = g.GangPacker()
    rows = []
    try:
        for seed, (n, n_rows, n_pods, big) in enumerate([(10_000, 100_000, 300_000, 20), (50_000, 1_000_000, 1_000_000, 40)]):
            rows += reconcile_rows(p, args, seed, n, n_rows, n_pods, big)
        for seed, (n, n_pods, big) in enumerate([(10_000, 300_000, 20), (50_000, 1_000_000, 40)]):
            rows.append(marker_row(p, args, seed, n, n_pods, big))
    finally:
        p.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": c, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
