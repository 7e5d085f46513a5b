#!/usr/bin/env python
"""Drain every instance group's FIFO queue with tightly-pack / distribute-evenly from the reservations, three ways:
  (one)    gp_prepare_cluster_groups + gp_pack_batch(FIFO): two calls, nothing on the host between;
  (recipe) gp_build_availability -> gp_potential_nodes per instance group (its sub-table) -> gp_set_snapshot -> gp_pack_batch;
  (rounds) per instance group, gp_prepare_cluster on its sub-table + gp_pack_batch.
Workload: 10 000 synth nodes in 16 instance groups of unequal size (the cluster of prepare_zones_groups_bench.py), 100 000
reservations, and the fifo-da-50k queue round-robin over the instance groups.  Both packers in both FIFO modes.  Wall clock
around calls that end in a stream synchronise, the three paths alternated, rep 0 a warm-up.  The prepare call is also timed
alone.  The three paths must agree bit for bit (drivers, ExecutorNodes, availability left behind).  Prints one JSON line
with the card's name and power limit.  Needs a GPU."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from prepare_zones_groups_bench import ROOT, card, cluster, sort_args, sub_table  # noqa: E402,F401

import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import synth  # noqa: E402

ALGOS = {"tightly-pack": g.native.TIGHTLY_PACK, "distribute-evenly": g.native.DISTRIBUTE_EVENLY}
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "young")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10000)
    ap.add_argument("--groups", type=int, default=16)
    ap.add_argument("--apps", type=int, default=50000)
    ap.add_argument("--reservations", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    G = args.groups
    alloc, over, rnode, res, sort, ig = cluster(args.nodes, G, args.reservations)
    members = [np.nonzero(ig == i)[0] for i in range(G)]
    subs = [sub_table(alloc, over, rnode, res, sort, m) for m in members]
    apps = synth.make_apps(args.apps, groups=G, da_sweep=True)
    a = {k: np.asarray(apps[k]) for k in KEYS}
    a["group"] = np.asarray(apps["group"], np.int32)
    sel = [np.nonzero(a["group"] == i)[0] for i in range(G)]
    sub_apps = [{k: a[k][s] for k in KEYS} for s in sel]
    one, rec, rnd = g.GangPacker(), g.GangPacker(), g.GangPacker()
    i32 = lambda v: np.asarray(v, np.int32)
    rows = []
    for name, algo in ALGOS.items():
        for mode in (1, 2):
            def prepare():
                return one.prepare_cluster_groups(alloc, over, rnode, res, ig, G, *sort_args(sort), orders=False)

            def run_one():
                prepare()
                return one.pack_batch(a, algo, mode), one.get_snapshot()

            def run_recipe():
                av, _ = rec.build_availability(alloc, over, rnode, res)
                eo, do, eoff, doff = [], [], [0], [0]
                for i, m in enumerate(members):
                    d, e = rec.potential_nodes(av[0][m], av[1][m], *sort_args(subs[i][4]))
                    eo.append(m[e]); do.append(m[d])
                    eoff.append(eoff[-1] + len(e)); doff.append(doff[-1] + len(d))
                rec.set_snapshot(av[0], av[1], av[2], i32(np.concatenate(eo)), i32(np.concatenate(do)), i32(eoff), i32(doff))
                return rec.pack_batch(a, algo, mode), rec.get_snapshot()

            def run_rounds():
                outs, avail = [], [np.zeros(args.nodes, np.int64) for _ in range(3)]
                for i, m in enumerate(members):
                    rnd.prepare_cluster(*subs[i][:4], *sort_args(subs[i][4]))
                    outs.append(rnd.pack_batch(sub_apps[i], algo, mode))
                    for k, x in enumerate(rnd.get_snapshot()):
                        avail[k][m] = x
                return outs, avail

            # bit-equality of the three paths (ExecutorNodes compared where the driver was placed)
            (drv, exe, off), snap = run_one()
            (d2, e2, o2), snap2 = run_recipe()
            agree = bool(np.array_equal(drv, d2) and np.array_equal(off, o2))
            agree &= all(np.array_equal(exe[off[j]:off[j + 1]], e2[o2[j]:o2[j + 1]]) for j in np.nonzero(drv >= 0)[0])
            agree &= all(np.array_equal(x, y) for x, y in zip(snap, snap2))
            outs, avail3 = run_rounds()
            for i, m in enumerate(members):
                s = sel[i]
                d3, e3, o3 = outs[i]
                agree &= bool(np.array_equal(drv[s], np.where(d3 >= 0, m[np.maximum(d3, 0)], d3)))
                for j in np.nonzero(d3 >= 0)[0]:
                    agree &= bool(np.array_equal(exe[off[s[j]]:off[s[j] + 1]], m[e3[o3[j]:o3[j + 1]]]))
                agree &= all(np.array_equal(x[m], y[m]) for x, y in zip(snap, avail3))
            t = {"prepare": [], "one": [], "recipe": [], "rounds": []}
            for r in range(args.reps + 1):
                t0 = time.perf_counter(); prepare(); t1 = time.perf_counter()
                run_one(); t2 = time.perf_counter()
                run_recipe(); t3 = time.perf_counter()
                run_rounds(); t4 = time.perf_counter()
                if r:
                    t["prepare"].append(t1 - t0); t["one"].append(t2 - t1); t["recipe"].append(t3 - t2); t["rounds"].append(t4 - t3)
            med = {k: round(float(np.median(v)) * 1e3, 3) for k, v in t.items()}
            rows.append({"algo": name, "mode": mode, "prepare_ms": med["prepare"], "prepare_ms_min": round(min(t["prepare"]) * 1e3, 3),
                         "one_ms": med["one"], "one_ms_min": round(min(t["one"]) * 1e3, 3), "recipe_ms": med["recipe"],
                         "rounds_ms": med["rounds"], "placed": int((drv >= 0).sum()), "paths_agree": agree})
    for p in (one, rec, rnd):
        p.close()
    print(json.dumps({"workload": "%d nodes in %d instance groups of unequal size, %d reservations, fifo-da queue of %d applications"
                                  % (args.nodes, G, args.reservations, args.apps), "reps": args.reps,
                      "card": card(), "paths_agree": all(r["paths_agree"] for r in rows), "results": rows}))


if __name__ == "__main__":
    main()
