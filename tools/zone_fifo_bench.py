#!/usr/bin/env python
"""fitEarlierDrivers with single-az-tightly-pack: ONE launch (gp_pack_fifo_zones) against the per-driver call sequence it
replaces (gp_pack_batch_zones for one application + gp_reserve_placements(subtract), exact accounting so that both run the
same arithmetic).  3 000 nodes in 3 zones, a queue of 2 000 drivers; host buffers in, host results out, wall clock.
Prints one JSON line; the two paths must agree bit for bit.

--packer az-aware-tightly-pack: ONE launch (gp_pack_fifo_az_aware) against the per-driver sequence of two contexts -- one
holds the zone-grouped snapshot and runs gp_pack_batch_zones for the driver, the other the undivided snapshot and runs
gp_pack_one when no zone wins; both are charged with gp_reserve_placements(subtract) after every placed driver.  3 000
nodes in 4 zones of unequal size; every 250th application asks for more executors than the largest zone holds, so the
undivided fallback runs (the JSON line reports how often and how many it placed).

--packer az-aware-tightly-pack --independent: a batch of independent decisions on the same cluster, one
gp_pack_batch_az_aware call against the two-context recipe it replaces -- gp_pack_batch_zones on a context holding the
zone-grouped snapshot, the zone -1 applications gathered on the host, gp_pack_batch(tightly-pack) over the undivided
orders on a second context, the results merged on the host.  Both snapshots stay resident (no upload is timed); every
50th application asks for more executors than the largest zone holds.  The two paths must agree bit for bit, and the
JSON line names the card and its power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import synth  # noqa: E402


def az_case(q, big_every):
    """3 000 nodes in 4 zones of unequal size and q synth applications, every big_every-th larger than any zone holds."""
    n = 3000
    nodes = synth.make_nodes(n)
    cpu, mem, gpu = nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"]
    order = synth.priority_order(cpu, mem).astype(np.int32)
    share = np.array([0.45, 0.3, 0.17, 0.08])                          # zones of unequal size
    Z = len(share)
    zone_of = np.searchsorted(np.cumsum(share), (np.arange(n) * 0.6180339887) % 1.0, side="right").clip(0, Z - 1)
    eo = np.concatenate([order[zone_of[order] == z] for z in range(Z)]).astype(np.int32)
    eoff = np.concatenate([[0], np.cumsum([(zone_of == z).sum() for z in range(Z)])]).astype(np.int32)
    apps = synth.make_apps(q, seed=11)
    a = {k: np.array(apps[k]) for k in KEYS}
    a["young"] = np.ones(q, np.uint8)
    for i in range(0, q, big_every):                                    # larger than any one zone holds
        caps = np.minimum(np.maximum(cpu, 0) // max(int(a["exe_cpu"][i]), 1), np.maximum(mem, 0) // max(int(a["exe_mem"][i]), 1))
        a["count"][i] = int(max(caps[zone_of == z].sum() for z in range(Z)) * 1.1) + 1
    return n, Z, cpu, mem, gpu, order, eo, eoff, a


KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")


def card():
    """name and power limit of the card, read in the same run as the measurement"""
    import torch
    import subprocess
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": out}


def az_aware_independent():
    q, reps = 4000, 20
    n, Z, cpu, mem, gpu, order, eo, eoff, a = az_case(q, 50)
    sc, sm, sg = cpu + 4000, mem + (8 << 30), gpu
    p, pz, pu = g.GangPacker(), g.GangPacker(), g.GangPacker()
    p.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)                   # every zone a candidate: no trailing group
    p.set_schedulable(sc, sm, sg)
    pz.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
    pz.set_schedulable(sc, sm, sg)
    pu.set_snapshot(cpu, mem, gpu, order, order)

    def one_call():
        return p.pack_batch_az_aware(a, order, order, Z)

    def recipe():
        zone, drv, exe, off, avg = pz.pack_batch_zones(a, 0)
        fb = np.nonzero(zone == -1)[0]
        if fb.size:
            d2, e2, o2 = pu.pack_batch({k: a[k][fb] for k in KEYS}, 0, 0)
            drv[fb] = d2
            for j in np.nonzero(d2 >= 0)[0]:
                i = fb[j]
                exe[off[i]:off[i + 1]] = e2[o2[j]:o2[j + 1]]
        return zone, drv, exe, off, avg

    t_one, t_two = [], []
    for r in range(reps + 2):                                           # alternate the two paths; the first two are warm-up
        for f, ts in ((one_call, t_one), (recipe, t_two)):
            t0 = time.perf_counter()
            res = f()
            if r >= 2:
                ts.append(time.perf_counter() - t0)
        if r == 0:
            got, want = one_call(), recipe()
            fallbacks = p.stats()["scan_path_apps"]
    zone, gd, ge, goff, avg = got
    placed = np.zeros(len(ge), bool)
    for i in np.nonzero(gd >= 0)[0]:
        placed[goff[i]:goff[i + 1]] = True
    won = zone >= 0
    same = bool(np.array_equal(zone, want[0]) and np.array_equal(gd, want[1]) and np.array_equal(ge[placed], want[2][placed])
                and np.array_equal(avg[won].view(np.uint64), want[4][won].view(np.uint64)) and (avg[~won] == 0.0).all())
    del res
    print(json.dumps(dict({"workload": "az-aware-tightly-pack, %d independent decisions, %d nodes in %d zones of unequal size"
                                       % (q, n, Z),
                           "one_call_ms": float(np.median(t_one)) * 1e3, "one_call_ms_min": float(np.min(t_one)) * 1e3,
                           "two_context_recipe_ms": float(np.median(t_two)) * 1e3,
                           "two_context_recipe_ms_min": float(np.min(t_two)) * 1e3, "reps": reps,
                           "placed": int((gd >= 0).sum()), "fallback_ran": int(fallbacks),
                           "fallback_placed": int(((zone == -1) & (gd >= 0)).sum()), "paths_agree": same}, **card())))
    for x in (p, pz, pu):
        x.close()


def az_aware():
    q, q_loop = 2000, 300
    n, Z, cpu, mem, gpu, order, eo, eoff, a = az_case(q, 250)
    keys = KEYS
    sc, sm, sg = cpu + 4000, mem + (8 << 30), gpu
    p, pz, pu = g.GangPacker(), g.GangPacker(), g.GangPacker()

    def fresh():
        p.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
        p.set_schedulable(sc, sm, sg)

    ts = []
    for _ in range(5):
        fresh()
        t0 = time.perf_counter()
        zone, gd, ge, goff, _ = p.pack_fifo_az_aware(a, 2, order, order, Z)
        ts.append(time.perf_counter() - t0)
    fallbacks = p.stats()["scan_path_apps"]
    one_launch_ms = float(np.min(ts[1:])) * 1e3
    # the per-driver sequence on the first q_loop drivers
    pz.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
    pz.set_schedulable(sc, sm, sg)
    pu.set_snapshot(cpu, mem, gpu, order, order)
    t0 = time.perf_counter()
    ld = np.full(q_loop, -9, np.int32)
    lex = []
    for i in range(q_loop):
        one = {k: a[k][i:i + 1] for k in keys}
        _, d1, e1, o1, _ = pz.pack_batch_zones(one, 0)
        if d1[0] < 0:
            has, d, en = pu.pack_one(0, (one["drv_cpu"][0], one["drv_mem"][0], one["drv_gpu"][0]),
                                     (one["exe_cpu"][0], one["exe_mem"][0], one["exe_gpu"][0]), int(one["count"][0]))
            d1 = np.array([d if has else -1], np.int32); e1 = np.asarray(en, np.int32)
        ld[i] = d1[0]
        lex.append(e1.copy() if d1[0] >= 0 else None)
        if d1[0] >= 0:
            placed = (d1, e1, o1)
            pz.reserve_placements(one, placed, subtract=True)
            pu.reserve_placements(one, placed, subtract=True)
    loop_ms = (time.perf_counter() - t0) * 1e3
    same = bool(np.array_equal(ld, gd[:q_loop]))
    for i in range(q_loop):
        if gd[i] >= 0:
            same = same and bool(np.array_equal(lex[i], ge[goff[i]:goff[i + 1]]))
    print(json.dumps({"workload": "az-aware-tightly-pack under FIFO, %d nodes in %d zones of unequal size, queue of %d drivers "
                                  "(exact accounting)" % (n, Z, q),
                      "one_launch_ms": one_launch_ms, "one_launch_us_per_driver": one_launch_ms * 1e3 / q,
                      "placed": int((gd >= 0).sum()), "fallback_ran": int(fallbacks),
                      "fallback_placed": int(((zone == -1) & (gd >= 0)).sum()),
                      "fallback_ran_in_sample": int((zone[:q_loop] == -1).sum()),
                      "per_driver_calls_us_per_driver": loop_ms * 1e3 / q_loop, "per_driver_sample": q_loop, "paths_agree": same}))
    for x in (p, pz, pu):
        x.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packer", choices=("single-az-tightly-pack", "az-aware-tightly-pack"), default="single-az-tightly-pack")
    ap.add_argument("--independent", action="store_true", help="az-aware-tightly-pack: a batch of independent decisions")
    args = ap.parse_args()
    if args.independent and args.packer != "az-aware-tightly-pack":
        ap.error("--independent goes with --packer az-aware-tightly-pack")
    if args.packer == "az-aware-tightly-pack":
        return az_aware_independent() if args.independent else az_aware()
    n, Z, q, q_loop = 3000, 3, 2000, 300
    nodes = synth.make_nodes(n)
    cpu, mem, gpu = nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"]
    order = synth.priority_order(cpu, mem)
    zone_of = np.arange(n) % Z
    eo = np.concatenate([order[zone_of[order] == z] for z in range(Z)]).astype(np.int32)
    eoff = np.concatenate([[0], np.cumsum([(zone_of == z).sum() for z in range(Z)])]).astype(np.int32)
    apps = synth.make_apps(q, seed=11)
    keys = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
    a = {k: apps[k] for k in keys}
    a["young"] = np.ones(q, np.uint8)
    p = g.GangPacker()
    sc, sm, sg = cpu + 4000, mem + (8 << 30), gpu

    def fresh():
        p.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
        p.set_schedulable(sc, sm, sg)

    ts = []
    for _ in range(5):
        fresh()
        t0 = time.perf_counter()
        zone, gd, ge, goff, _ = p.pack_fifo_zones(a, 0, 2)
        ts.append(time.perf_counter() - t0)
    one_launch_ms = float(np.min(ts[1:])) * 1e3
    # the per-driver sequence on the first q_loop drivers
    fresh()
    t0 = time.perf_counter()
    ld = np.full(q_loop, -9, np.int32)
    lex = []
    for i in range(q_loop):
        one = {k: a[k][i:i + 1] for k in keys}
        z1, d1, e1, o1, _ = p.pack_batch_zones(one, 0)
        ld[i] = d1[0]
        lex.append(e1.copy() if d1[0] >= 0 else np.full(int(a["count"][i]), -9, np.int32))
        if d1[0] >= 0:
            p.reserve_placements(one, (d1, e1, o1), subtract=True)
    loop_ms = (time.perf_counter() - t0) * 1e3
    same = bool(np.array_equal(ld, gd[:q_loop]))
    for i in range(q_loop):
        if gd[i] >= 0:
            same = same and bool(np.array_equal(lex[i], ge[goff[i]:goff[i + 1]]))
    print(json.dumps({"workload": "single-az-tightly-pack under FIFO, %d nodes in %d zones, queue of %d drivers (exact accounting)" % (n, Z, q),
                      "one_launch_ms": one_launch_ms, "one_launch_us_per_driver": one_launch_ms * 1e3 / q,
                      "placed": int((gd >= 0).sum()), "per_driver_calls_us_per_driver": loop_ms * 1e3 / q_loop,
                      "per_driver_sample": q_loop, "paths_agree": same}))
    p.close()


if __name__ == "__main__":
    main()
