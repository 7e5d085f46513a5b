"""One simulated driver Predicate with the resident driver table against today's per-call FIFO queue.

  table arm:  the driver-table flush of the pod events since the last Predicate, then gp_pack_fifo_driver_table (the queue
              selected, ordered and packed on the device)
  today:      the host's filterToEarliestAndSort over the pending drivers, shouldSkipDriverFifo and the gp_apps columns, then
              gp_pack_batch in GP_MODE_FIFO_REFERENCE (the columns uploaded)

Both arms run on one context over the same snapshot (re-uploaded, untimed, before each arm) and are timed alternately with a
host clock around work that ends in the entries' own synchronise.  Before every pair, `churn` of the pending drivers are
added, changed or deleted.  The requesting driver is the newest of a random instance group, so its queue holds about
1/16 of the pending drivers.  The "today" arm is a Python restatement of the per-call recipe (string-level
filter_to_earliest_and_sort over dicts, starting from parsed resources): its host time measures a Python host layer, not the
Go scheduler's sort.Slice over listed pods.  Every timed pair's queue, driver nodes, offsets and the
ExecutorNodes of placed drivers are compared.  H2D bytes are counted from the arrays each arm hands the library.

    python tools/resident_queue_bench.py --out results.json [--drivers 10000 50000] [--nodes 10000] [--churn 0.01] [--reps 30]
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
from k8s_spark_scheduler_b200 import drivers  # noqa: E402
from oracle.pyref import filter_to_earliest_and_sort  # noqa: E402

SEC = 10 ** 9
GROUPS = [f"ig-{i}" for i in range(16)]
DEFAULT_AGE = 300 * SEC


def resources(rng):
    return {"drv": [int(rng.integers(1, 4)) * 1000, int(rng.integers(1, 8)) << 30, 0],
            "exe": [int(rng.integers(1, 4)) * 1000, int(rng.integers(1, 8)) << 30, 0], "min": int(rng.integers(1, 8))}


class Cluster:
    """The pending drivers as a pod lister holds them (string level, listed in slot order) and as the driver table holds them"""

    def __init__(self, rng, n):
        self.rng = rng
        self.table = drivers.DriverTable(n_slots=2 * n, n_groups=len(GROUPS), n_schedulers=1)
        self.pods = {}
        self.n = 0
        for _ in range(n):
            self.add()

    def add(self):
        uid = f"driver-{self.n}"
        self.n += 1
        self.set(uid)

    def set(self, uid):
        r = self.rng
        p = dict(uid=uid, created=int(r.integers(0, 7200)) * SEC, scheduler="spark-scheduler", group=GROUPS[r.integers(len(GROUPS))],
                 node=None, res=resources(r))
        self.pods[uid] = p
        self.table.set_driver(uid, p["created"], p["scheduler"], p["group"], p["res"])

    def churn(self, k):
        live = list(self.pods)
        for _ in range(k):
            op = self.rng.random()
            if op < 0.4:
                self.add()
            elif op < 0.7:
                uid = live[self.rng.integers(len(live))]
                if uid in self.pods:
                    del self.pods[uid]
                    self.table.delete_driver(uid)
            else:
                uid = live[self.rng.integers(len(live))]
                if uid in self.pods:
                    self.set(uid)

    def requesting(self):
        grp = GROUPS[self.rng.integers(len(GROUPS))]
        return max((p for p in self.pods.values() if p["group"] == grp), key=lambda p: (p["created"], p["uid"]))


def today_apps(cl, me, now):
    """filterToEarliestAndSort over the listed drivers (slot order: the lister's order in this simulation), then the gp_apps
    columns with shouldSkipDriverFifo; the requesting driver last"""
    listed = sorted(cl.pods.values(), key=lambda p: cl.table.slot_of(p["uid"]))
    queue = filter_to_earliest_and_sort(me, listed) + [me]
    q = len(queue)
    apps = {k: np.empty(q, np.int64) for k in drivers.QUANTITIES}
    for j, p in enumerate(queue):
        for k, v in zip(drivers.QUANTITIES, p["res"]["drv"] + p["res"]["exe"]):
            apps[k][j] = v
    apps["count"] = np.array([p["res"]["min"] for p in queue], np.int32)
    apps["young"] = np.array([p["created"] + DEFAULT_AGE > now for p in queue[:-1]] + [False], np.uint8)
    apps["group"] = np.zeros(q, np.int32)
    apps["off"] = np.zeros(q + 1, np.int64)
    np.cumsum(apps["count"], out=apps["off"][1:])
    return [cl.table.slot_of(p["uid"]) for p in queue], apps


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
    name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
    return dict(name=name, power_limit=limit)


def run(p, n_drivers, n_nodes, churn, reps, seed):
    rng = np.random.default_rng(seed)
    snap = (rng.integers(8, 65, n_nodes) * 1000, rng.integers(32, 257, n_nodes).astype(np.int64) << 30, np.zeros(n_nodes, np.int64),
            np.arange(n_nodes, dtype=np.int32), np.arange(n_nodes, dtype=np.int32))
    cl = Cluster(rng, n_drivers)
    cl.table.flush(p)
    now = 7000 * SEC
    t_flush, t_table, t_host, t_pack, agree, h2d_t, h2d_h, queued = [], [], [], [], 0, [], [], []
    for rep in range(reps + 2):                       # the first two pairs warm up
        cl.churn(max(1, int(churn * n_drivers)))
        me = cl.requesting()
        order = (0, 1) if rep % 2 == 0 else (1, 0)
        res = {}
        for arm in order:
            p.set_snapshot(*snap)
            if arm == 0:
                t0 = time.perf_counter()
                d = cl.table.delta()
                if d["reset"] is not None:
                    p.driver_table_reset(**d["reset"])
                p.driver_table_update(d)
                cl.table.mirror.apply(d)
                t1 = time.perf_counter()
                q = dict(requesting_slot=cl.table.slot_of(me["uid"]), predicate_group=0, n_slots=cl.table.size["n_slots"],
                         enforce_after_ns=cl.table.group_ages(DEFAULT_AGE), now=now)
                got = p.pack_fifo_driver_table(q, g.native.TIGHTLY_PACK, g.native.MODE_FIFO_REFERENCE)
                t2 = time.perf_counter()
                res[0] = got
                if rep >= 2:
                    t_flush.append(t1 - t0); t_table.append(t2 - t1)
                    h2d_t.append(sum(v.nbytes for v in d.values() if isinstance(v, np.ndarray)) + q["enforce_after_ns"].nbytes)
            else:
                t0 = time.perf_counter()
                slots, apps = today_apps(cl, me, now)
                t1 = time.perf_counter()
                drv, exe, off = p.pack_batch(apps, g.native.TIGHTLY_PACK, g.native.MODE_FIFO_REFERENCE)
                t2 = time.perf_counter()
                res[1] = (slots, drv, exe, off)
                if rep >= 2:
                    t_host.append(t1 - t0); t_pack.append(t2 - t1)
                    h2d_h.append(sum(v.nbytes for v in apps.values()))
        got, (slots, drv, exe, off) = res[0], res[1]
        ok = (got["queue_slot"].tolist() == slots and np.array_equal(got["driver_node"], drv) and np.array_equal(got["off"], off)
              and all(np.array_equal(got["executor_nodes"][off[i]:off[i + 1]], exe[off[i]:off[i + 1]]) for i in np.flatnonzero(drv >= 0)))
        if rep >= 2:
            agree += int(ok)
            queued.append(len(slots))
    ms = lambda xs: round(float(np.median(xs)) * 1e3, 3)
    tot_t = [a + b for a, b in zip(t_flush, t_table)]
    tot_h = [a + b for a, b in zip(t_host, t_pack)]
    return dict(n_drivers=n_drivers, n_nodes=n_nodes, churn=churn, pairs=reps, agreeing_pairs=agree, median_queue=int(np.median(queued)),
                ms=dict(table_total=ms(tot_t), table_flush=ms(t_flush), table_entry=ms(t_table),
                        today_total=ms(tot_h), today_host_queue=ms(t_host), today_pack_batch=ms(t_pack)),
                h2d_bytes=dict(table=int(np.median(h2d_t)), today=int(np.median(h2d_h))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--drivers", type=int, nargs="+", default=[10_000, 50_000])
    ap.add_argument("--nodes", type=int, default=10_000)
    ap.add_argument("--churn", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    g.native.load()
    p = g.GangPacker()
    result = dict(card=card(), rows=[])
    try:
        for n in a.drivers:
            r = run(p, n, a.nodes, a.churn, a.reps, seed=n)
            result["rows"].append(r)
            print(json.dumps(r))
    finally:
        p.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
