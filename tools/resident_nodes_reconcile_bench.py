"""The failover reconciler and the unschedulable-pod marker over the resident node table, against today's resident calls.

  reconcile, node table:  the label, node, reservation and overhead table flushes, then gp_reconcile_find_nodes_node_table
                          (per listed node: its node-table, reservation-table and overhead-table ids)
  reconcile, today:       the label, reservation and overhead table flushes, the host's decoding of every node's instance
                          group from its label mirror, then gp_reconcile_find_nodes_resident with allocatable, group,
                          creation and both flags uploaded per node
  marker, node table:     gp_exceeds_cluster_capacity_node_table / gp_exceeds_cluster_capacity_affinity_node_table
  marker, today:          the host's decoding of every node's zone, then gp_exceeds_cluster_capacity_resident /
                          gp_exceeds_cluster_capacity_affinity_label_table with allocatable and zone uploaded per node

Two contexts are fed the same seeded node-event stream (allocatable, readiness, creation and label changes of `churn` of the
nodes, plus as many reservation rewrites).  Each pair of calls is timed alternately, with a host clock around work that ends
in the entries' own synchronise, and every timed pair's results are compared.  H2D bytes per call are those of the per-node
columns and of the deltas, counted from the arrays (the drivers are the same on both sides and not counted).  The overhead
table holds no pod records here: its flush is the same empty update on both sides.

    python tools/resident_nodes_reconcile_bench.py --out results.json [--nodes 10000 50000] [--churn 0.01] [--reps 30]
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
GROUPS = [f"ig-{i}" for i in range(16)]
IG = "instance-group"
ROWS_PER_NODE = 10
STALE, MARKER = 200, 1000
AFFS = [{"required": [{"matchExpressions": [(IG, "In", GROUPS[4 * k:4 * k + 4])]}]} for k in range(4)]


class Side:
    """One context and its host tables"""

    def __init__(self, n, node_table):
        self.p = g.GangPacker()
        self.labels = affinity.LabelTable(n_node_ids=n, n_keys=8, n_values=64)
        self.table = nodes.NodeTable(self.labels, n_node_ids=n) if node_table else None
        self.p.reservation_table_reset(n_slots=n * ROWS_PER_NODE, n_node_ids=n)
        self.p.overhead_table_reset(n_slots=1, n_node_ids=n, n_app_keys=1, n_app_ids=1, n_names=1)
        self.alloc = np.zeros((3, n), np.int64)
        self.flags = np.zeros((2, n), np.uint8)
        self.creation = np.zeros(n, np.int64)
        self.bytes = 0

    def event(self, name, i, lab, alloc, uns, rdy, cre):
        self.labels.set_node(name, lab)
        self.alloc[:, i] = alloc
        self.flags[:, i] = (uns, rdy)
        self.creation[i] = cre
        if self.table is not None:
            self.table.set_node(name, alloc, uns, rdy, creation=cre)

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
    lab = {nodes.ZONE_LABEL: ZONES[rng.integers(len(ZONES))]}
    if rng.random() < 0.95:
        lab[IG] = GROUPS[rng.integers(len(GROUPS))]
    return lab


def equal(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(equal(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and np.array_equal(a, b)
    return a == b


def defined(r):
    """a reconcile result with the executor-node entries past placed[i] (undefined) set to -1"""
    placed, execn, off, avail = r
    keep = np.full(len(execn), -1, np.int32)
    for i, k in enumerate(placed):
        keep[off[i]:off[i] + max(int(k), 0)] = execn[off[i]:off[i] + max(int(k), 0)]
    return placed, keep, off, avail


def run(n, churn, reps, warmup, seed=1):
    rng = np.random.default_rng(seed)
    names = [f"node-{rng.integers(1 << 40):012x}-{i}" for i in range(n)]
    old, new = Side(n, False), Side(n, True)

    def apply(ix):
        for i in ix:
            lab = node_labels(rng)
            alloc = (int(rng.integers(8, 65)) * 1000, int(rng.integers(32, 513)) << 30, int(rng.integers(0, 9)))
            uns, rdy = bool(rng.random() < 0.02), bool(rng.random() < 0.98)
            cre = int(rng.integers(0, 1 << 20)) * 10 ** 9
            for s in (old, new):
                s.event(names[i], i, lab, alloc, uns, rdy, cre)

    def res_delta(k):
        slot = rng.choice(n * ROWS_PER_NODE, k, replace=False).astype(np.int32)
        return dict(slot=slot, node_id=rng.integers(0, n, k).astype(np.int32), cpu_milli=rng.integers(0, 4000, k),
                    mem_bytes=rng.integers(0, 8 << 30, k), gpu=rng.integers(0, 2, k))

    apply(range(n))
    first = res_delta(n * ROWS_PER_NODE // 2)
    for s in (old, new):
        s.flush(first)
    rid = np.arange(n, dtype=np.int32)
    oid = np.full(n, -1, np.int32)
    k = max(1, int(round(churn * n)))
    arms = ("reconcile", "marker", "marker_affinity")
    times = {a: {"node_table": [], "today": []} for a in arms}
    bytes_ = {a: {"node_table": [], "today": []} for a in arms}
    agree = {a: 0 for a in arms}
    for it in range(warmup + reps):
        apply(rng.choice(n, k, replace=False))
        rd = res_delta(k)
        ra = nodes.reconcile_label_args(new.labels, IG, GROUPS)
        G, miss = ra["n_groups"], ra["instance_group_missing"]
        za = nodes.label_args(new.labels, zones=ZONES)
        zk = dict(zone_key=za["zone_key"], n_zones=za["n_zones"], zone_value=za["zone_value"], zone_missing=za["zone_missing"])
        stale = dict(exe_cpu=rng.integers(1, 9, STALE) * 1000, exe_mem=rng.integers(1, 17, STALE) * (1 << 30),
                     exe_gpu=np.zeros(STALE, np.int64), count=rng.integers(0, 5, STALE).astype(np.int32),
                     group=rng.integers(0, G, STALE).astype(np.int32))
        mk = dict(drv_cpu=rng.integers(1, 5, MARKER) * 1000, drv_mem=rng.integers(1, 9, MARKER) * (1 << 30),
                  drv_gpu=np.zeros(MARKER, np.int64), exe_cpu=rng.integers(1, 17, MARKER) * 1000,
                  exe_mem=rng.integers(1, 33, MARKER) * (1 << 30), exe_gpu=np.zeros(MARKER, np.int64),
                  count=rng.integers(0, 200, MARKER).astype(np.int32), group=np.full(MARKER, -1, np.int32))
        amk = dict(mk, group=rng.integers(0, len(AFFS), MARKER).astype(np.int32))
        enc = new.labels.encode_affinities(AFFS, names)
        packer = int(it % 5)

        def today(arm):
            s = old
            ids = s.labels.node_ids(names)
            if arm == "reconcile":
                s.flush(rd)
                grp = nodes.reconcile_groups(s.labels.mirror, ids, **ra)
                out = s.p.reconcile_find_nodes_resident(rid, tuple(s.alloc), None, grp, s.creation, stale, G, unschedulable=s.flags[0],
                                                        ready=s.flags[1], overhead_node_id=oid)
                return out, n * (24 + 4 + 8 + 1 + 1 + 4 + 4) + s.bytes
            zone = nodes.label_columns(s.labels.mirror, ids, **zk)["zone_id"]
            if arm == "marker":
                return (s.p.exceeds_cluster_capacity_resident(tuple(s.alloc), oid, mk, packer, zone_id=zone, n_zones=zk["n_zones"]),
                        n * (24 + 4 + 4))
            return (s.p.exceeds_cluster_capacity_affinity_label_table(tuple(s.alloc), oid, ids, enc, amk, packer, zone_id=zone,
                                                                      n_zones=zk["n_zones"]), n * (24 + 4 + 4 + 4))

        def node_table(arm):
            s = new
            nd = dict(node_table_id=s.table.node_ids(names), reservation_id=rid, overhead_node_id=oid, **zk)
            if arm == "reconcile":
                s.flush(rd)
                nd = dict(nd, node_table_id=s.table.node_ids(names), zone_key=-1, n_zones=1, zone_value=None, zone_missing=-1,
                          instance_group_key=ra["instance_group_key"], instance_group_value=ra["instance_group_value"])
                return s.p.reconcile_find_nodes_node_table(nd, stale, G, miss), n * 12 + s.bytes
            if arm == "marker":
                return s.p.exceeds_cluster_capacity_node_table(nd, mk, packer), n * 8
            return s.p.exceeds_cluster_capacity_affinity_node_table(nd, enc, amk, packer), n * 8

        for arm in arms:
            res = {}
            for side in (("today", "node_table") if it % 2 else ("node_table", "today")):
                t0 = time.perf_counter()
                out, b = (today if side == "today" else node_table)(arm)
                dt = time.perf_counter() - t0
                res[side] = out
                if it >= warmup:
                    times[arm][side].append(dt * 1e3)
                    bytes_[arm][side].append(b)
            if arm == "reconcile":
                res = {k: defined(v) for k, v in res.items()}
            if not equal(res["today"], res["node_table"]):
                raise AssertionError(f"n={n} churn={churn} iteration {it} {arm}: the two calls disagree")
            agree[arm] += it >= warmup
    for s in (old, new):
        s.p.close()
    stat = lambda v: dict(median=float(np.median(v)), p10=float(np.percentile(v, 10)), p90=float(np.percentile(v, 90)))
    return dict(n_nodes=n, churn=churn, events_per_call=k, n_groups=len(GROUPS), stale_drivers=STALE, marker_drivers=MARKER,
                reps=reps, agreeing_pairs=agree,
                ms={a: {s: stat(v) for s, v in times[a].items()} for a in arms},
                h2d_bytes={a: {s: float(np.median(v)) for s, v in bytes_[a].items()} for a in arms})


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
    return dict(name=name, power_limit=limit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, nargs="+", default=[10000, 50000])
    ap.add_argument("--churn", type=float, nargs="+", default=[0.01])
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    result = dict(card=card(), runs=[run(n, c, a.reps, a.warmup) for n in a.nodes for c in a.churn])
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    for r in result["runs"]:
        print(json.dumps({k: r[k] for k in ("n_nodes", "churn", "ms", "h2d_bytes", "agreeing_pairs")}))


if __name__ == "__main__":
    main()
