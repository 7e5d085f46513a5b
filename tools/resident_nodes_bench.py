"""One simulated driver Predicate with the resident node table against today's resident Predicate.

  node table:  the label, node, reservation and overhead table flushes, then gp_prepare_cluster_groups_node_table
               (per listed node: its node-table, reservation-table and overhead-table ids, and is_driver_candidate)
  today:       the label, reservation and overhead table flushes, the host's decoding of the per-call columns (allocatable,
               flags, zone, instance group, label ranks) and the argsort of the node names, then
               gp_prepare_cluster_groups_resident

Two contexts are fed the same seeded node-event stream (allocatable, readiness and label changes of `churn` of the nodes, plus
as many reservation rewrites) and are timed alternately, one Predicate each, with a host clock around work that ends in the
entries' own synchronise.  Every timed pair's orders, counts, ties and snapshot are compared.  H2D bytes per Predicate are
those of the per-call columns and of the deltas, counted from the arrays.  The overhead table holds no pod records here: its
flush is the same empty update on both sides.

    python tools/resident_nodes_bench.py --out results.json [--nodes 10000 50000] [--churn 0.001 0.01] [--reps 40]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import affinity, nodes  # noqa: E402

ZONES = [f"zone-{i}" for i in range(3)]
GROUPS = [f"ig-{i}" for i in range(4)]
PRIORITY = ["hi", "mid", "lo"]
ROWS_PER_NODE = 10


class Side:
    """One context and its host tables"""

    def __init__(self, n, node_table):
        self.p = g.GangPacker()
        self.labels = affinity.LabelTable(n_node_ids=n, n_keys=8, n_values=64)
        self.table = nodes.NodeTable(self.labels, n_node_ids=n) if node_table else None
        self.n = n
        self.p.reservation_table_reset(n_slots=n * ROWS_PER_NODE, n_node_ids=n)
        self.p.overhead_table_reset(n_slots=1, n_node_ids=n, n_app_keys=1, n_app_ids=1, n_names=1)
        self.alloc = np.zeros((3, n), np.int64)
        self.flags = np.zeros((2, n), np.uint8)
        self.bytes = 0

    def event(self, name, i, lab, alloc, uns, rdy):
        self.labels.set_node(name, lab)
        self.alloc[:, i] = alloc
        self.flags[:, i] = (uns, rdy)
        if self.table is not None:
            self.table.set_node(name, alloc, uns, rdy)

    def flush(self, res_delta):
        d = self.labels.delta()
        self.bytes = sum(v.nbytes for k, v in d.items() if isinstance(v, np.ndarray))
        if d["reset"] is not None:
            self.p.label_table_reset(**d["reset"])
        self.p.label_table_update(d)
        self.labels.mirror.apply(d)
        if self.table is not None:
            d = self.table.delta()
            self.bytes += sum(v.nbytes for k, v in d.items() if isinstance(v, np.ndarray))
            if d["reset"] is not None:
                self.p.node_table_reset(**d["reset"])
            self.p.node_table_update(d)
            self.table.mirror.apply(d)
        self.p.reservation_table_update(res_delta)
        self.bytes += sum(v.nbytes for v in res_delta.values())
        self.p.overhead_table_update({})


def node_labels(rng):
    lab = {nodes.ZONE_LABEL: ZONES[rng.integers(len(ZONES))], "instance-group": GROUPS[rng.integers(len(GROUPS))]}
    if rng.random() < 0.7:
        lab["priority"] = PRIORITY[rng.integers(len(PRIORITY))]
    return lab


def run(n, churn, reps, warmup, seed=1):
    rng = np.random.default_rng(seed)
    names = [f"node-{rng.integers(1 << 40):012x}-{i}" for i in range(n)]
    old, new = Side(n, False), Side(n, True)

    def apply(ix):
        for i in ix:
            lab = node_labels(rng)
            alloc = (int(rng.integers(8, 65)) * 1000, int(rng.integers(32, 513)) << 30, int(rng.integers(0, 9)))
            uns, rdy = bool(rng.random() < 0.02), bool(rng.random() < 0.98)
            for s in (old, new):
                s.event(names[i], i, lab, alloc, uns, rdy)

    def res_delta(k):
        slot = rng.choice(n * ROWS_PER_NODE, k, replace=False).astype(np.int32)
        return dict(slot=slot, node_id=rng.integers(0, n, k).astype(np.int32), cpu_milli=rng.integers(0, 4000, k),
                    mem_bytes=rng.integers(0, 8 << 30, k), gpu=rng.integers(0, 2, k))

    apply(range(n))
    first = res_delta(n * ROWS_PER_NODE // 2)
    for s in (old, new):
        s.flush(first)
    order_ids = np.arange(n)
    k = max(1, int(round(churn * n)))
    cand = np.ones(n, np.uint8)
    times = {"node_table": [], "today": []}
    bytes_ = {"node_table": [], "today": []}
    agree = 0
    for it in range(warmup + reps):
        apply(rng.choice(n, k, replace=False))
        rd = res_delta(k)
        args = nodes.label_args(new.labels, zones=ZONES, instance_group_label="instance-group", instance_groups=GROUPS,
                                driver_priority=("priority", PRIORITY), executor_priority=("priority", PRIORITY))
        res = {}
        for side in (("today", "node_table") if it % 2 else ("node_table", "today")):
            t0 = time.perf_counter()
            if side == "today":
                s = old
                s.flush(rd)
                ids = s.labels.node_ids(names)
                lab = nodes.label_columns(s.labels.mirror, ids, **args)
                rank = np.empty(n, np.int32)
                rank[np.argsort(np.array(names))] = np.arange(n, dtype=np.int32)
                rid = order_ids.astype(np.int32)
                oid = np.full(n, -1, np.int32)
                out = s.p.prepare_cluster_groups_resident(rid, tuple(s.alloc), None, lab["instance_group"], len(GROUPS), lab["zone_id"],
                                                          args["n_zones"], rank, cand, s.flags[0], s.flags[1], lab["driver_label_rank"],
                                                          lab["executor_label_rank"], overhead_node_id=oid)
                call_bytes = n * (24 + 4 + 4 + 4 + 8 + 1 + 1 + 1 + 4 + 4)
            else:
                s = new
                s.flush(rd)
                nd = dict(node_table_id=s.table.node_ids(names), reservation_id=order_ids.astype(np.int32),
                          overhead_node_id=np.full(n, -1, np.int32), is_driver_candidate=cand, **args)
                out = s.p.prepare_cluster_groups_node_table(nd, None, len(GROUPS))
                call_bytes = n * 13
            dt = time.perf_counter() - t0
            res[side] = (out, s.p.get_snapshot())
            if it >= warmup:
                times[side].append(dt * 1e3)
                bytes_[side].append(call_bytes + s.bytes)
        a, b = res["today"], res["node_table"]
        ok = all(np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y for x, y in zip(a[1], b[1]))
        ok = ok and all(np.array_equal(a[0][key], b[0][key]) if isinstance(a[0][key], np.ndarray) else a[0][key] == b[0][key]
                        for key in a[0])
        if not ok:
            raise AssertionError(f"n={n} churn={churn} iteration {it}: the two Predicates disagree")
        agree += it >= warmup
    for s in (old, new):
        s.p.close()
    stat = lambda v: dict(median=float(np.median(v)), p10=float(np.percentile(v, 10)), p90=float(np.percentile(v, 90)))
    return dict(n_nodes=n, churn=churn, events_per_predicate=k, reps=reps, agreeing_pairs=agree,
                ms={k: stat(v) for k, v in times.items()}, h2d_bytes={k: float(np.median(v)) for k, v in bytes_.items()})


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
    return dict(name=name, power_limit=limit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, nargs="+", default=[10000, 50000])
    ap.add_argument("--churn", type=float, nargs="+", default=[0.001, 0.01])
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    result = dict(card=card(), runs=[run(n, c, a.reps, a.warmup) for n in a.nodes for c in a.churn])
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    for r in result["runs"]:
        print(json.dumps({k: r[k] for k in ("n_nodes", "churn", "ms", "h2d_bytes", "agreeing_pairs")}))


if __name__ == "__main__":
    main()
