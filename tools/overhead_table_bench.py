"""Time the resident overhead table (gp_overhead_table_update + gp_overhead_table_query) against gp_node_overhead.

    python tools/overhead_table_bench.py [--reps 10] [--warmup 2] [--out FILE]

Clusters: overhead.synthetic_cluster as in tools/overhead_bench.py -- 10 000 nodes x 300 000 pod records and 50 000 x
1 000 000 -- loaded into an overhead.OverheadTable and sent to the device as one delta.  Then simulated Predicates, for a
churn of 0.1 % and of 1 % of the records per Predicate: that many pods deleted and re-added on another node (their slots
rewritten), plus one new ResourceReservation of 20 pods.  Per Predicate, alternating in the same run:
  resident     one gp_overhead_table_update with the Predicate's delta and one gp_overhead_table_query over every node (the
               per-node sums and n_warned; has_reservation is not asked for), wall clock around each (each ends in a stream
               synchronise)
  per-call     gp_node_overhead over the same state's arrays (overhead.to_encoding of the numpy mirror), from ordinary
               (pageable) numpy arrays and from page-locked ones (GangPacker.pinned); as in tools/overhead_bench.py these
               calls also return has_reservation
Every timed resident answer is checked equal to both per-call answers.  Medians over --reps Predicates after --warmup, with
the 10th and 90th percentiles.  Twenty further queries and one further update under torch.profiler (CUDA activities) give
the H2D / kernel / D2H device time per call, with the share of the expected kernel launches the trace holds (below 1: the
capture dropped events and the split is not to be used); bytes each way are computed from the shapes.  The deltas and
encodings are built before the timed loop and not timed.  Prints the card's name and power limit, read in the same run.  Needs a GPU."""
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

ARRAYS = ("node_id", "req_cpu_milli", "req_mem_bytes", "req_gpu", "listed", "app_key", "app_id", "name_id", "is_executor",
          "spark_scheduler", "rr_app_key", "rr_pod_off", "rr_pod_name", "soft_app_id", "soft_pod_off", "soft_pod_name", "node_ids")
DELTA = ("slot", "node_id", "req_cpu_milli", "req_mem_bytes", "req_gpu", "listed", "app_key", "app_id", "name_id", "is_executor",
         "spark_scheduler", "rr_app_key", "rr_exists", "member_kind", "member_app", "member_name", "member_present")


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


def split(fn, prefixes, launches, calls=20):
    """-> (H2D ms, kernel ms, D2H ms) per call, averaged over `calls` calls in one torch.profiler trace, and the share of the
    expected kernel launches (`launches` per call) the trace holds: below 1 means it dropped events"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
        torch_sync()
    h2d = ker = d2h = 0.0
    seen = 0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if "HtoD" in e.key:
            h2d += t
        elif "DtoH" in e.key:
            d2h += t
        elif any(p in e.key for p in prefixes):
            ker += t
            seen += e.count
    return [round(x / 1e3 / calls, 4) for x in (h2d, ker, d2h)], round(seen / (launches * calls), 3)


def torch_sync():
    import torch
    torch.cuda.synchronize()


def churn_delta(table, pods, nodes, rng, frac, tag):
    """one Predicate's worth of events -> its delta"""
    for i in rng.choice(len(pods), max(1, int(len(pods) * frac)), replace=False):
        p = pods[i]
        table.delete(p)
        q = dict(p, uid=f"{p['uid']}-{tag}", nodeName=nodes[rng.integers(len(nodes))])
        table.add(q)
        pods[i] = q
    table.rr_set((f"ns-{tag % 16}", f"bench-{tag}"), [f"bench-{tag}-exec-{e}" for e in range(20)])
    return table.delta()


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a[0] + a[1], b[0] + b[1])) and a[-1] == b[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    p = g.GangPacker()
    rows = []
    try:
        for seed, (n, q, big) in enumerate([(10_000, 300_000, 20), (50_000, 1_000_000, 40)]):
            nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(seed, n, q, big_apps=big, big_executors=2000)
            table = oh.OverheadTable(n_slots=q, n_node_ids=n, n_app_keys=1 << 16, n_app_ids=1 << 16, n_names=1 << 21)
            mirror = oh.TableMirror()
            for pod in pods:
                table.add(pod)
            for pod in lister.values():
                table.lister_set(pod)
            for k, v in rrs.items():
                table.rr_set(k, v)
            for k, v in soft.items():
                table.soft_set(k, v)
            d = table.delta()
            mirror.apply(d)
            p.overhead_table_reset(**d["reset"])
            t_load, _ = clock(lambda: p.overhead_table_update(d))
            ids = table.node_ids(nodes)
            assert (ids >= 0).all()
            rng = np.random.default_rng(seed)
            for frac in (0.001, 0.01):
                steps = []
                for s in range(args.warmup + args.reps):
                    dl = churn_delta(table, pods, nodes, rng, frac, int(frac * 1e4) * 1000 + s)
                    mirror.apply(dl)
                    steps.append((dl, oh.to_encoding(mirror, ids)))
                pin = {k: p.pinned(max(len(e[k]) for _, e in steps) or 1, steps[0][1][k].dtype) for k in ARRAYS}
                t = {k: [] for k in ("update", "query", "predicate", "per_call_pageable", "per_call_pinned")}
                for s, (dl, enc) in enumerate(steps):
                    t_up, _ = clock(lambda: p.overhead_table_update(dl))
                    t_q, got = clock(lambda: p.overhead_table_query(ids, has_reservation=False))
                    t_pg, want = clock(lambda: p.node_overhead(enc))
                    pinned = dict(enc)
                    for k in ARRAYS:
                        pinned[k] = pin[k][:len(enc[k])]
                        pinned[k][...] = enc[k]
                    t_pn, want2 = clock(lambda: p.node_overhead(pinned))
                    assert same(got, want) and same(got, want2), "resident and per-call answers disagree"
                    if s >= args.warmup:
                        for k, v in zip(t, (t_up, t_q, t_up + t_q, t_pg, t_pn)):
                            t[k].append(v)
                _, _, has, _ = p.overhead_table_query(ids)
                assert np.array_equal(has[:len(table.slots)], want[2][:len(table.slots)])
                # the query launches gp_oh_dir, gp_oh_pods and gp_oh_finish
                q_split, q_seen = split(lambda: p.overhead_table_query(ids, has_reservation=False), ("gp_oh_",), 3)
                # one update with a Predicate's delta launches gp_oht_check, gp_oht_apply and gp_oht_insert
                probe = churn_delta(table, pods, nodes, rng, frac, 999_000 + int(frac * 1e4))
                mirror.apply(probe)
                u_split, u_seen = split(lambda: p.overhead_table_update(probe), ("gp_oht_",), 3, calls=1)
                assert same(p.overhead_table_query(ids, has_reservation=False), p.node_overhead(oh.to_encoding(mirror, ids)))
                up_bytes = [sum(dl[k].nbytes for k in DELTA) for dl, _ in steps[args.warmup:]]
                row = dict(nodes=n, pod_records=q, churn_fraction=frac, slot_writes_per_update=int(np.median([len(dl["slot"]) for dl, _ in steps])),
                           member_writes_per_update=int(np.median([len(dl["member_kind"]) for dl, _ in steps])),
                           initial_load_update_ms=round(t_load, 3),
                           ms={k: stats(v) for k, v in t.items()},
                           query_split_ms_h2d_kernels_d2h=q_split, query_split_launches_seen=q_seen,
                           update_split_ms_h2d_kernels_d2h=u_split, update_split_launches_seen=u_seen,
                           query_h2d_bytes=4 * n, query_d2h_bytes=48 * n + 16,
                           update_h2d_bytes_median=int(np.median(up_bytes)), update_d2h_bytes=24,
                           per_call_h2d_bytes=int(np.median([sum(e[k].nbytes for k in ARRAYS) for _, e in steps])),
                           per_call_d2h_bytes=48 * n + q + 16, parity_checked_calls=len(steps) + 1)
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
