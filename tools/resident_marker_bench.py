"""One simulated unschedulable-pod marker scan with the resident driver table against today's per-call recipe.

  table arm:  the driver-table flush of the pod events since the last scan, then gp_exceeds_cluster_capacity_driver_table
              (stale selection, order, columns and the capacity checks on the device)
  today:      the host's stale filter over the pending drivers (spark-scheduler, creation + timeout < now), the interning and
              encoding of their distinct required affinities, the gp_apps columns, then
              gp_exceeds_cluster_capacity_affinity_node_table (the columns uploaded)

Both arms run on one context over the same node, label and (empty) overhead tables and are timed alternately, with a host
clock around work that ends in the entries' own synchronise.  Before every pair, `churn` of the pending drivers are added,
changed or deleted; about half of them are stale.  The "today" arm starts from parsed resources and is a Python
restatement of the host recipe: its host time measures a Python host layer, not the Go scheduler's.  Every timed pair's
stale drivers, exceeds and affinity-error flags are compared.  H2D bytes are counted from the arrays each arm hands the
library (the per-node id columns, the programs, and the driver delta or the gp_apps columns).

    python tools/resident_marker_bench.py --out results.json [--nodes 10000 50000] [--drivers 10000 50000] [--reps 30]
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
from k8s_spark_scheduler_b200 import affinity, drivers, nodes  # noqa: E402

SEC = 10 ** 9
ZONES = [f"zone-{i}" for i in range(3)]
GROUPS = [f"ig-{i}" for i in range(16)]
IG = "instance-group"
SCHEDULER = "spark-scheduler"
TIMEOUT, NOW = 600 * SEC, 7200 * SEC
# 16 distinct required affinities: four groups of instance groups, each alone, in one zone or in all but one zone
AFFS = ([{"nodeSelector": None, "required": [{"matchExpressions": [(IG, "In", GROUPS[4 * k:4 * k + 4])]}]} for k in range(4)] +
        [{"nodeSelector": {IG: GROUPS[k]}, "required": None} for k in range(6)] +
        [{"nodeSelector": {nodes.ZONE_LABEL: z}, "required": [{"matchExpressions": [(IG, "In", GROUPS[:8])]}]} for z in ZONES] +
        [{"nodeSelector": None, "required": [{"matchExpressions": [(nodes.ZONE_LABEL, "NotIn", [z])]}]} for z in ZONES])
PACKERS = {"tightly-pack": 0, "single-az-tightly-pack": 3}


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
    return dict(name=name, power_limit=limit)


class Cluster:
    """The pending drivers as a pod lister holds them (parsed) and as the driver table holds them, over n labelled nodes"""

    def __init__(self, p, rng, n_nodes, n_drivers):
        self.p, self.rng = p, rng
        self.labels = affinity.LabelTable(n_node_ids=n_nodes, n_keys=8, n_values=64)
        self.nodes = nodes.NodeTable(self.labels, n_node_ids=n_nodes)
        self.names = [f"node-{i}" for i in range(n_nodes)]
        for name in self.names:
            lab = {nodes.ZONE_LABEL: ZONES[rng.integers(len(ZONES))]}
            if rng.random() < 0.95:
                lab[IG] = GROUPS[rng.integers(len(GROUPS))]
            self.labels.set_node(name, lab)
            self.nodes.set_node(name, (int(rng.integers(8, 65)) * 1000, int(rng.integers(32, 513)) << 30, int(rng.integers(0, 9))),
                                False, True)
        self.labels.flush(p)
        self.nodes.flush(p)
        p.overhead_table_reset(n_slots=1, n_node_ids=n_nodes, n_app_keys=1, n_app_ids=1, n_names=1)
        self.table = drivers.DriverTable(n_slots=2 * n_drivers, n_groups=len(GROUPS), n_schedulers=2)
        self.pods = {}
        self.n = 0
        for _ in range(n_drivers):
            self.add()
        self.nd = dict(node_table_id=self.nodes.node_ids(self.names), overhead_node_id=np.zeros(n_nodes, np.int32) - 1,
                       **nodes.label_args(self.labels, zones=ZONES, zone_label=nodes.ZONE_LABEL, instance_group_label=IG,
                                          instance_groups=GROUPS))

    def add(self):
        uid = f"driver-{self.n}"
        self.n += 1
        self.set(uid)

    def set(self, uid):
        r = self.rng
        res = {"drv": [int(r.integers(1, 4)) * 1000, int(r.integers(1, 8)) << 30, 0],
               "exe": [int(r.integers(1, 9)) * 1000, int(r.integers(1, 33)) << 30, int(r.random() < 0.1)], "min": int(r.integers(1, 40))}
        pod = dict(uid=uid, created=int(r.integers(0, 2 * (NOW - TIMEOUT) // SEC)) * SEC,
                   scheduler=SCHEDULER if r.random() < 0.95 else "other", res=res,
                   affinity=None if r.random() < 0.1 else AFFS[r.integers(len(AFFS))])
        self.pods[uid] = pod
        self.table.set_driver(uid, pod["created"], pod["scheduler"], GROUPS[r.integers(len(GROUPS))], res, affinity=pod["affinity"])

    def churn(self, k):
        live = list(self.pods)
        for _ in range(k):
            op = self.rng.random()
            if op < 0.4:
                self.add()
            else:
                uid = live[self.rng.integers(len(live))]
                if uid not in self.pods:
                    continue
                if op < 0.7:
                    del self.pods[uid]
                    self.table.delete_driver(uid)
                else:
                    self.set(uid)


def today(cl, packer):
    """the host recipe: the stale filter, the distinct affinities interned and encoded, the gp_apps columns, one call"""
    stale = [pd for pd in cl.pods.values() if pd["scheduler"] == SCHEDULER and pd["created"] + TIMEOUT < NOW]
    ids, progs = {}, []
    group = np.empty(len(stale), np.int32)
    for j, pd in enumerate(stale):
        k = drivers.affinity_key(pd["affinity"])
        if k not in ids:
            ids[k] = len(progs)
            progs.append(pd["affinity"] or drivers.MATCH_ALL)
        group[j] = ids[k]
    enc = cl.labels.encode_affinities(progs, cl.names)
    apps = {k: np.array([pd["res"]["drv" if j < 3 else "exe"][j % 3] for pd in stale], np.int64) for j, k in enumerate(drivers.QUANTITIES)}
    apps["count"] = np.array([pd["res"]["min"] for pd in stale], np.int32)
    apps["group"] = group
    exceeds, err = cl.p.exceeds_cluster_capacity_affinity_node_table(cl.nd, enc, apps, packer)
    h2d = sum(v.nbytes for v in apps.values()) + sum(v.nbytes for v in enc.values() if isinstance(v, np.ndarray))
    return [pd["uid"] for pd in stale], exceeds, err, h2d


def run(p, n_nodes, n_drivers, packer, churn, reps, seed):
    rng = np.random.default_rng(seed)
    cl = Cluster(p, rng, n_nodes, n_drivers)
    cl.table.flush(p)
    node_bytes = sum(v.nbytes for v in cl.nd.values() if isinstance(v, np.ndarray))
    t_flush, t_table, t_today, agree, h2d_t, h2d_h, n_stale = [], [], [], 0, [], [], []
    for rep in range(reps + 2):                       # the first two pairs warm up
        cl.churn(max(1, int(churn * n_drivers)))
        res = {}
        for arm in ((0, 1) if rep % 2 == 0 else (1, 0)):
            if arm == 0:
                t0 = time.perf_counter()
                d = cl.table.delta()
                cl.table.push(p, d)
                cl.table.mirror.apply(d)
                enc = cl.labels.encode_affinities(cl.table.affinity_programs(), cl.names)
                t1 = time.perf_counter()
                got = p.exceeds_cluster_capacity_driver_table(cl.nd, enc, cl.table.scheduler_id(SCHEDULER), TIMEOUT, NOW, packer,
                                                              cap=n_drivers * 2)
                t2 = time.perf_counter()
                res[0] = got
                if rep >= 2:
                    t_flush.append(t1 - t0); t_table.append(t2 - t1)
                    h2d_t.append(node_bytes + sum(v.nbytes for v in d.values() if isinstance(v, np.ndarray)) +
                                 sum(v.nbytes for v in enc.values() if isinstance(v, np.ndarray)))
            else:
                t0 = time.perf_counter()
                uids, exceeds, err, h2d = today(cl, packer)
                t1 = time.perf_counter()
                res[1] = (uids, exceeds, err)
                if rep >= 2:
                    t_today.append(t1 - t0)
                    h2d_h.append(node_bytes + h2d)
        got, (uids, exceeds, err) = res[0], res[1]
        by_slot = {cl.table.slot_of(u): (int(e), int(a)) for u, e, a in zip(uids, exceeds, err)}
        ok = (sorted(by_slot) == sorted(got["stale_slot"].tolist()) and
              all(by_slot[int(s)] == ((int(e) if o == 0 else int(by_slot[int(s)][0])), int(o == 1))
                  for s, e, o in zip(got["stale_slot"], got["exceeds"], got["outcome"])) and not (got["outcome"] == 2).any())
        if rep >= 2:
            agree += int(ok)
            n_stale.append(len(uids))
    ms = lambda xs: dict(median=round(float(np.median(xs)) * 1e3, 3), p10=round(float(np.percentile(xs, 10)) * 1e3, 3),
                         p90=round(float(np.percentile(xs, 90)) * 1e3, 3))
    tot_t = [a + b for a, b in zip(t_flush, t_table)]
    return dict(n_nodes=n_nodes, n_drivers=n_drivers, packer=[k for k, v in PACKERS.items() if v == packer][0], churn=churn,
                pairs=reps, agreeing_pairs=agree, median_stale=int(np.median(n_stale)), distinct_affinities=len(AFFS),
                ms=dict(table_total=ms(tot_t), table_flush_and_programs=ms(t_flush), table_entry=ms(t_table), today_total=ms(t_today)),
                h2d_bytes=dict(table=int(np.median(h2d_t)), today=int(np.median(h2d_h))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--nodes", type=int, nargs="+", default=[10_000, 50_000])
    ap.add_argument("--drivers", type=int, nargs="+", default=[10_000, 50_000])
    ap.add_argument("--packers", nargs="+", default=list(PACKERS))
    ap.add_argument("--churn", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    g.native.load()
    result = dict(card=card(), rows=[])
    for n in a.nodes:
        for q in a.drivers:
            for name in a.packers:
                p = g.GangPacker()
                try:
                    r = run(p, n, q, PACKERS[name], a.churn, a.reps, seed=n + q)
                finally:
                    p.close()
                result["rows"].append(r)
                print(json.dumps(r), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
