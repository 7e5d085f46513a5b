"""Time gp_exceeds_cluster_capacity -- the unschedulable-pod marker's whole sweep in one device call -- against the recipes it
replaces, on the same clusters and drivers.

    python tools/capacity_check_bench.py [--reps 10] [--warmup 2] [--out FILE]

Clusters: N = 10 000 and 50 000 nodes in 16 affinity classes x 8 zones; Q = 1 000, 10 000 and 100 000 stale drivers of
1-32 executors, spread over the classes, a share of them with executors no node can hold.  For each point and packer:
  new            one gp_exceeds_cluster_capacity call (tightly-pack, single-az-tightly-pack, az-aware-tightly-pack)
  tightly-pack   gp_set_snapshot with one instance group per class, then one gp_pack_batch_wire (64-bit quantities, 16-bit
                 ExecutorNodes) over all drivers: the whole placement comes back and is thrown away
  single-az      per class: gp_set_snapshot with the class's zones as groups + gp_set_schedulable + gp_pack_batch_zones
  az-aware       per class: the same snapshot + gp_pack_batch_az_aware with the undivided orders
Wall clock (time.perf_counter) around each complete recipe; every call ends in a stream synchronise.  Both sides run through
the Python binding with their inputs marshalled beforehand.  The answers of each recipe are checked against the new call.
Prints the card's name and power limit with the numbers.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import k8s_spark_scheduler_b200 as g  # noqa: E402

G = 1 << 30
CLASSES, ZONES = 16, 8


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def cluster(rng, n):
    alloc = [rng.integers(8, 97, n) * 1000, rng.integers(32, 385, n) * G, (rng.integers(0, 8, n) == 0) * 4]
    over = [np.full(n, 500), np.full(n, G), np.zeros(n)]
    zone = rng.integers(0, ZONES, n).astype(np.int32)
    group = rng.integers(0, CLASSES, n).astype(np.int32)
    return [np.asarray(x, np.int64) for x in alloc], [np.asarray(x, np.int64) for x in over], zone, group


def drivers(rng, q):
    big = rng.random(q) < 0.3                                  # executors larger than any node: these drivers exceed
    return {"drv_cpu": rng.integers(1, 5, q).astype(np.int64) * 1000, "drv_mem": rng.integers(1, 9, q).astype(np.int64) * G,
            "drv_gpu": np.zeros(q, np.int64),
            "exe_cpu": rng.integers(1, 9, q).astype(np.int64) * 1000,
            "exe_mem": np.where(big, 512 * G, rng.integers(1, 33, q) * G).astype(np.int64),
            "exe_gpu": np.zeros(q, np.int64), "count": rng.integers(1, 33, q).astype(np.int32),
            "group": rng.integers(0, CLASSES, q).astype(np.int32)}


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    rows = []
    p = g.GangPacker()
    try:
        for n in (10_000, 50_000):
            rng = np.random.default_rng(n)
            alloc, over, zone, group = cluster(rng, n)
            sched = [alloc[d] - over[d] for d in range(3)]
            # per-class orders (lister order: any), and per class the zone groups with the undivided order restricted to them
            orders = [rng.permutation(np.nonzero(group == c)[0]).astype(np.int32) for c in range(CLASSES)]
            off = np.zeros(CLASSES + 1, np.int32)
            off[1:] = np.cumsum([len(o) for o in orders])
            flat = np.concatenate(orders)
            zoned = []
            for o in orders:
                zs = list(dict.fromkeys(zone[o].tolist()))
                parts = [o[zone[o] == z] for z in zs]
                zoff = np.zeros(len(parts) + 1, np.int32)
                zoff[1:] = np.cumsum([len(x) for x in parts])
                zoned.append((np.concatenate(parts), zoff, o, len(zs)))
            for q in (1_000, 10_000, 100_000):
                apps = drivers(rng, q)
                sel = [np.nonzero(apps["group"] == c)[0] for c in range(CLASSES)]
                subs = [{k: v[s] for k, v in apps.items()} for s in sel]
                total = int(apps["count"].sum())
                out = (np.empty(q, np.int32), np.empty(total, np.uint16))
                wire = dict(quantity_bits=64, node_bits=16)
                row = {"nodes": n, "drivers": q, "exceeding": None}

                def new(name):
                    return p.exceeds_cluster_capacity(alloc, apps, g.native.BINPACKERS[name], overhead=over, zone_id=zone, n_zones=ZONES,
                                                      node_group=group, n_groups=CLASSES)

                def old_tightly():
                    p.set_snapshot(*sched, flat, flat, off, off)
                    return p.pack_batch(apps, g.TIGHTLY_PACK, out=out, wire=wire)[0] < 0

                def old_zones(az_aware):
                    res = np.empty(q, bool)
                    for c in range(CLASSES):
                        order, zoff, undivided, nz = zoned[c]
                        p.set_snapshot(*sched, order, order, zoff, zoff)
                        p.set_schedulable(*sched)
                        if az_aware:
                            res[sel[c]] = p.pack_batch_az_aware(subs[c], undivided, undivided, nz)[1] < 0
                        else:
                            res[sel[c]] = p.pack_batch_zones(subs[c], g.TIGHTLY_PACK)[0] < 0
                    return res

                for name, old in (("tightly-pack", old_tightly), ("single-az-tightly-pack", lambda: old_zones(False)),
                                  ("az-aware-tightly-pack", lambda: old_zones(True))):
                    want = new(name)
                    assert np.array_equal(want.astype(bool), old()), (n, q, name)
                    row["exceeding"] = int(want.sum())
                    tn = timed(lambda: new(name), args.reps, args.warmup)
                    to = timed(old, args.reps, args.warmup)
                    row[name] = {"new_ms_median": float(np.median(tn)), "new_ms_best": float(np.min(tn)),
                                 "old_ms_median": float(np.median(to)), "old_ms_best": float(np.min(to))}
                rows.append(row)
                print(json.dumps(row), flush=True)
    finally:
        p.close()
    result = {"card": card(), "points": rows}
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
