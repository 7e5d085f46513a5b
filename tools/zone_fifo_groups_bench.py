#!/usr/bin/env python
"""fitEarlierDrivers of 16 instance groups with a zone-aware packer: ONE gp_pack_fifo_zones_groups launch (one CTA per
instance group) against the two ways to drain the same queues with the single-group entry points:
  (a) the recipe without it: 16 rounds of gp_set_snapshot + gp_set_schedulable + gp_pack_fifo_zones / gp_pack_fifo_az_aware
      on one context, every round timed with its upload;
  (b) 16 resident contexts, one per instance group, each with its snapshot already uploaded (no upload timed).
10 000 synth nodes in 16 instance groups of unequal size, 3 or 4 zones of unequal size each; the queue is the fifo-da-50k
one (50 000 dynamic-allocation applications round-robin over the groups, none young, so a queue blocks at its first
driver that fits nowhere).  Every packer in both accounting modes.  The three paths must agree bit for bit (drivers, local
zones, ExecutorNodes, averages, availability).  Prints one JSON line, with the card's name and power limit."""
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

PACKERS = {"single-az-tightly-pack": g.native.BP_SINGLE_AZ_TIGHTLY_PACK,
           "single-az-minimal-fragmentation": g.native.BP_SINGLE_AZ_MINIMAL_FRAGMENTATION,
           "az-aware-tightly-pack": g.native.BP_AZ_AWARE_TIGHTLY_PACK}
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "young")


def card():
    """name and power limit of the card, read in the same run as the measurement"""
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": out}


def cluster(n, G):
    """-> cpu, mem, gpu, per instance group (its nodes, undivided priority order, zone-grouped order and offsets)"""
    nodes = synth.make_nodes(n)
    cpu, mem, gpu = nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"]
    w = np.arange(1, G + 1, dtype=np.float64)                           # instance groups of unequal size (1 : 2 : ... : G)
    owner = np.searchsorted(np.cumsum(w / w.sum()), (np.arange(n) * 0.6180339887) % 1.0, side="right").clip(0, G - 1)
    groups = []
    for i in range(G):
        members = np.nonzero(owner == i)[0]
        Z = 3 + i % 2
        share = np.array([0.4, 0.3, 0.2, 0.1][:Z]); share /= share.sum()   # zones of unequal size
        zone = np.searchsorted(np.cumsum(share), (np.arange(len(members)) * 0.7548776662) % 1.0, side="right").clip(0, Z - 1)
        zone_of = dict(zip(members.tolist(), zone.tolist()))
        order = synth.priority_order(cpu, mem, members)
        zorder = np.concatenate([[v for v in order if zone_of[int(v)] == z] for z in range(Z)]).astype(np.int32)
        zoff = np.concatenate([[0], np.cumsum([(zone == z).sum() for z in range(Z)])]).astype(np.int32)
        groups.append(dict(nodes=members, order=order, zorder=zorder, zoff=zoff, Z=Z))
    return cpu, mem, gpu, groups


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10000)
    ap.add_argument("--groups", type=int, default=16)
    ap.add_argument("--apps", type=int, default=50000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    G = args.groups
    cpu, mem, gpu, groups = cluster(args.nodes, G)
    sc, sm, sg = cpu + 4000, mem + (8 << 30), gpu
    apps = synth.make_apps(args.apps, groups=G, da_sweep=True)
    a = {k: np.asarray(apps[k]) for k in KEYS}
    a["group"] = np.asarray(apps["group"], np.int32)
    sel = [np.nonzero(a["group"] == i)[0] for i in range(G)]
    sub = [{k: a[k][s] for k in KEYS} for s in sel]
    # the whole snapshot: instance group after instance group, its zones as groups
    eo = np.concatenate([x["zorder"] for x in groups]).astype(np.int32)
    base = np.cumsum([0] + [len(x["zorder"]) for x in groups])
    eoff = np.concatenate([[0]] + [b + x["zoff"][1:] for b, x in zip(base, groups)]).astype(np.int32)
    goff = np.cumsum([0] + [x["Z"] for x in groups]).astype(np.int32)
    one, rec, res = g.GangPacker(), g.GangPacker(), [g.GangPacker() for _ in range(G)]
    rows = []
    for name, pid in PACKERS.items():
        az = pid == g.native.BP_AZ_AWARE_TIGHTLY_PACK
        kw = dict(group_off=goff)
        if az:
            kw.update(n_zones=np.array([x["Z"] for x in groups], np.int32), exec_off=base.astype(np.int32),
                      exec_order=np.concatenate([x["order"] for x in groups]).astype(np.int32), drv_off=base.astype(np.int32),
                      drv_order=np.concatenate([x["order"] for x in groups]).astype(np.int32))
        for mode in (1, 2):
            def single(p, i):
                x = groups[i]
                if az:
                    return p.pack_fifo_az_aware(sub[i], mode, x["order"], x["order"], x["Z"])
                return p.pack_fifo_zones(sub[i], 0 if pid == g.native.BP_SINGLE_AZ_TIGHTLY_PACK else 2, mode)

            def load_one():
                one.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
                one.set_schedulable(sc, sm, sg)

            def load_resident():
                for i, p in enumerate(res):
                    x = groups[i]
                    p.set_snapshot(cpu, mem, gpu, x["zorder"], x["zorder"], x["zoff"], x["zoff"])
                    p.set_schedulable(sc, sm, sg)

            def run_one():
                return one.pack_fifo_zones_groups(a, pid, mode, **kw)

            def run_recipe(keep=False):
                outs, snaps = [], []
                for i in range(G):
                    x = groups[i]
                    rec.set_snapshot(cpu, mem, gpu, x["zorder"], x["zorder"], x["zoff"], x["zoff"])
                    rec.set_schedulable(sc, sm, sg)
                    outs.append(single(rec, i))
                    if keep:
                        snaps.append(rec.get_snapshot())
                return outs, snaps

            def run_resident():
                return [single(p, i) for i, p in enumerate(res)]

            # bit-equality of the three paths
            load_one()
            zone, drv, exe, off, avg = run_one()
            snap = one.get_snapshot()
            fallbacks = one.stats()["scan_path_apps"]
            outs, snaps = run_recipe(keep=True)
            load_resident()
            outs_b = run_resident()
            agree = True
            for i in range(G):
                s = sel[i]
                for o in (outs[i], outs_b[i]):
                    z2, d2, e2, o2, v2 = o
                    agree &= bool(np.array_equal(zone[s], z2) and np.array_equal(drv[s], d2)
                                  and np.array_equal(avg[s].view(np.uint64), v2.view(np.uint64)))
                    for j in np.nonzero(d2 >= 0)[0]:
                        agree &= bool(np.array_equal(exe[off[s[j]]:off[s[j] + 1]], e2[o2[j]:o2[j + 1]]))
                for k in range(3):
                    agree &= bool(np.array_equal(snap[k][groups[i]["nodes"]], snaps[i][k][groups[i]["nodes"]]))
                    agree &= bool(np.array_equal(snap[k][groups[i]["nodes"]], res[i].get_snapshot()[k][groups[i]["nodes"]]))
            # timing: the three paths alternated, rep 0 is warm-up
            t = {"one": [], "a": [], "b": []}
            for r in range(args.reps + 1):
                load_one()
                t0 = time.perf_counter(); run_one(); t1 = time.perf_counter()
                run_recipe(); t2 = time.perf_counter()
                load_resident()
                t3 = time.perf_counter(); run_resident(); t4 = time.perf_counter()
                if r:
                    t["one"].append(t1 - t0); t["a"].append(t2 - t1); t["b"].append(t4 - t3)
            med = {k: float(np.median(v)) * 1e3 for k, v in t.items()}
            rows.append({"packer": name, "mode": mode, "one_launch_ms": med["one"], "one_launch_ms_min": min(t["one"]) * 1e3,
                         "recipe_a_ms": med["a"], "recipe_b_resident_ms": med["b"],
                         "recipe_b_resident_ms_min": min(t["b"]) * 1e3,
                         "speedup_vs_b": med["b"] / med["one"], "placed": int((drv >= 0).sum()),
                         "blocked": int((drv == -2).sum()), "fallback_ran": int(fallbacks) if az else None, "paths_agree": agree})
    for p in [one, rec] + res:
        p.close()
    print(json.dumps(dict({"workload": "%d nodes in %d instance groups of unequal size, 3-4 zones each, fifo-da queue of %d "
                                       "applications" % (args.nodes, G, args.apps), "reps": args.reps,
                           "paths_agree": all(r["paths_agree"] for r in rows), "results": rows}, **card())))


if __name__ == "__main__":
    main()
