#!/usr/bin/env python
"""Drain every instance group's zone-aware FIFO queue from the reservations, three ways:
  (one)    gp_prepare_cluster_zones_groups + gp_pack_fifo_zones_groups(groups == NULL): two calls, nothing on the host between;
  (recipe) gp_build_availability -> gp_potential_nodes per instance group (its sub-table) -> zone grouping in numpy ->
           gp_set_snapshot + gp_set_schedulable -> gp_pack_fifo_zones_groups with the explicit layout;
  (rounds) per instance group, gp_prepare_cluster_zones on its sub-table + gp_pack_fifo_zones / gp_pack_fifo_az_aware.
Workload: 10 000 synth nodes in 16 instance groups of unequal size, 3 or 4 zones each (zone names shared across instance
groups), 100 000 reservations, and the fifo-da-50k queue round-robin over the instance groups.  Every packer in both FIFO
modes.  Wall clock around calls that end in a stream synchronise, the three paths alternated, rep 0 a warm-up.  The prepare
call is also timed alone.  The three paths must agree bit for bit (drivers, local zones, ExecutorNodes, averages,
availability).  Prints one JSON line with the card's name and power limit.  Needs a GPU."""
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
from k8s_spark_scheduler_b200 import synth  # noqa: E402

N = g.native
PACKERS = {"single-az-tightly-pack": N.BP_SINGLE_AZ_TIGHTLY_PACK, "single-az-minimal-fragmentation": N.BP_SINGLE_AZ_MINIMAL_FRAGMENTATION,
           "az-aware-tightly-pack": N.BP_AZ_AWARE_TIGHTLY_PACK}
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "young")
GIB = 1 << 30


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def cluster(n, G, R, seed=5):
    """node table, reservations, sort columns and the instance group of every node"""
    rng = np.random.default_rng(seed)
    alloc = [rng.integers(8, 97, n) * 1000, rng.integers(32, 385, n) * GIB, np.zeros(n, np.int64)]
    over = [rng.integers(0, 3, n) * 250, rng.integers(0, 4, n) * (1 << 28), np.zeros(n, np.int64)]
    rnode = rng.integers(-1, n, R).astype(np.int32)
    res = [rng.integers(0, 6, R) * 500, rng.integers(0, 12, R) * (1 << 29), np.zeros(R, np.int64)]
    w = np.arange(1, G + 1, dtype=np.float64)                           # instance groups of unequal size (1 : 2 : ... : G)
    ig = np.searchsorted(np.cumsum(w / w.sum()), (np.arange(n) * 0.6180339887) % 1.0, side="right").clip(0, G - 1).astype(np.int32)
    zid = np.zeros(n, np.int32)
    for i in range(G):
        members = np.nonzero(ig == i)[0]
        Z = 3 + i % 2
        share = np.array([0.4, 0.3, 0.2, 0.1][:Z]); share /= share.sum()   # zones of unequal size
        zid[members] = np.searchsorted(np.cumsum(share), (np.arange(len(members)) * 0.7548776662) % 1.0, side="right").clip(0, Z - 1)
    sort = dict(zone_id=zid, n_zones=4, name_rank=np.argsort(rng.permutation(n)).astype(np.int32),
                is_driver_candidate=(rng.random(n) < 0.8).astype(np.uint8), unschedulable=(rng.random(n) < 0.05).astype(np.uint8),
                ready=(rng.random(n) < 0.95).astype(np.uint8))
    return alloc, over, rnode, res, sort, ig


def sub_table(alloc, over, rnode, res, sort, idx):
    pos = np.full(len(sort["zone_id"]), -1, np.int64)
    pos[idx] = np.arange(len(idx))
    rn = np.where(rnode >= 0, pos[np.maximum(rnode, 0)], -1).astype(np.int32)
    s = {k: v[idx] for k, v in sort.items() if k != "n_zones"}
    s["name_rank"] = np.argsort(np.argsort(sort["name_rank"][idx], kind="stable")).astype(np.int32)
    s["n_zones"] = sort["n_zones"]
    return [a[idx] for a in alloc], [o[idx] for o in over], rn, res, s


def sort_args(s):
    return (s["zone_id"], s["n_zones"], s["name_rank"], s["is_driver_candidate"], s["unschedulable"], s["ready"])


def group_by_zone(d, e, zid, az):
    """groupNodesByZone of one instance group's orders -> (exec_order, drv_order, exec_off, drv_off, n_zones)"""
    dz = zid[d]
    zones, first = np.unique(dz, return_index=True)
    cand = zones[np.isin(zones, zid[e])]
    cand = cand[np.argsort(first[np.isin(zones, zid[e])], kind="stable")]
    groups = [(e[zid[e] == z], d[zid[d] == z]) for z in cand]
    if az:
        te, td = e[~np.isin(zid[e], cand)], d[~np.isin(zid[d], cand)]
        if len(te) or len(td) or not len(cand):
            groups.append((te, td))
    elif not len(cand):
        groups.append((e[:0], d[:0]))
    eo = np.concatenate([x for x, _ in groups]) if groups else e[:0]
    do = np.concatenate([y for _, y in groups]) if groups else d[:0]
    eoff = np.cumsum([0] + [len(x) for x, _ in groups]); doff = np.cumsum([0] + [len(y) for _, y in groups])
    return eo, do, eoff, doff, len(cand)


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
    rows = []
    for name, pid in PACKERS.items():
        az = pid == N.BP_AZ_AWARE_TIGHTLY_PACK
        kind = N.LAYOUT_AZ_AWARE if az else N.LAYOUT_SINGLE_AZ
        for mode in (1, 2):
            def prepare():
                return one.prepare_cluster_zones_groups(alloc, over, rnode, res, ig, G, *sort_args(sort), kind=kind, layout=False)

            def run_one():
                prepare()
                return one.pack_fifo_zones_groups(a, pid, mode), one.get_snapshot()

            def run_recipe():
                av, sc = rec.build_availability(alloc, over, rnode, res)
                eo, do, eoff, doff, goff, nz, ue, ud = [], [], [0], [0], [0], [], [], []
                for i, m in enumerate(members):
                    d, e = rec.potential_nodes(av[0][m], av[1][m], *sort_args(subs[i][4]))
                    d, e = m[d], m[e]
                    x = group_by_zone(d, e, sort["zone_id"], az)
                    eoff += list(len(eo) + x[2][1:]); doff += list(len(do) + x[3][1:])
                    eo += list(x[0]); do += list(x[1]); goff.append(goff[-1] + len(x[2]) - 1); nz.append(x[4])
                    ue.append(e); ud.append(d)
                i32 = lambda v: np.asarray(v, np.int32)
                rec.set_snapshot(av[0], av[1], av[2], i32(eo), i32(do), i32(eoff), i32(doff))
                rec.set_schedulable(*sc)
                kw = dict(group_off=i32(goff))
                if az:
                    kw.update(n_zones=i32(nz), exec_off=i32(np.cumsum([0] + [len(x) for x in ue])), exec_order=i32(np.concatenate(ue)),
                              drv_off=i32(np.cumsum([0] + [len(x) for x in ud])), drv_order=i32(np.concatenate(ud)))
                return rec.pack_fifo_zones_groups(a, pid, mode, **kw), rec.get_snapshot()

            def run_rounds():
                outs, avail = [], [np.zeros(args.nodes, np.int64) for _ in range(3)]
                for i, m in enumerate(members):
                    s = subs[i]
                    rnd.prepare_cluster_zones(*s[:4], *sort_args(s[4]), kind=kind, layout=False)
                    o = rnd.pack_fifo_az_aware(sub_apps[i], mode) if az else \
                        rnd.pack_fifo_zones(sub_apps[i], 0 if pid == N.BP_SINGLE_AZ_TIGHTLY_PACK else 2, mode)
                    outs.append(o)
                    for k, x in enumerate(rnd.get_snapshot()):
                        avail[k][m] = x
                return outs, avail

            # bit-equality of the three paths
            (zone, drv, exe, off, avg), snap = run_one()
            (z2, d2, e2, o2, v2), snap2 = run_recipe()
            agree = bool(np.array_equal(zone, z2) and np.array_equal(drv, d2) and np.array_equal(off, o2)
                         and np.array_equal(exe, e2) and np.array_equal(avg.view(np.uint64), v2.view(np.uint64)))
            agree &= all(np.array_equal(x, y) for x, y in zip(snap, snap2))
            outs, avail3 = run_rounds()
            for i, m in enumerate(members):
                s = sel[i]
                z3, d3, e3, o3, v3 = outs[i]
                d3m = np.where(d3 >= 0, m[np.maximum(d3, 0)], d3)
                agree &= bool(np.array_equal(zone[s], z3) and np.array_equal(drv[s], d3m)
                              and np.array_equal(avg[s].view(np.uint64), v3.view(np.uint64)))
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
            rows.append({"packer": name, "mode": mode, "prepare_ms": med["prepare"], "prepare_ms_min": round(min(t["prepare"]) * 1e3, 3),
                         "one_ms": med["one"], "one_ms_min": round(min(t["one"]) * 1e3, 3), "recipe_ms": med["recipe"],
                         "rounds_ms": med["rounds"], "placed": int((drv >= 0).sum()), "paths_agree": agree})
    for p in (one, rec, rnd):
        p.close()
    print(json.dumps({"workload": "%d nodes in %d instance groups of unequal size, 3-4 zones each, %d reservations, fifo-da queue of %d "
                                  "applications" % (args.nodes, G, args.reservations, args.apps), "reps": args.reps,
                      "card": card(), "paths_agree": all(r["paths_agree"] for r in rows), "results": rows}))


if __name__ == "__main__":
    main()
