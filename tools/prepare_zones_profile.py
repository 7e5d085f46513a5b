#!/usr/bin/env python
"""Per-kernel device time and wall time of one gp_prepare_cluster_zones call, and of one gp_prepare_cluster_zones_groups call
where the package has it, from torch.profiler (diagnostic, not part of the bench contract).

    python tools/prepare_zones_profile.py [--calls 100] [--root TREE]

Workloads: the 10 000-node, 3-zone and 50 000-node, 8-zone points of prepare_zones_bench.py (100 000 reservations, both
layout kinds), and the 16-instance-group workload of prepare_zones_groups_bench.py (10 000 nodes, 100 000 reservations).
--root runs the package of another checkout (e.g. the parent commit, built) on the same inputs, for a before/after table.
Wall time: median over --calls calls without the profiler, after 20 warm-up calls.  Device time: the calls again under the
profiler, per kernel (and copy / memset) its launches per call and mean µs per call.  Prints one JSON line per workload,
each with the GPU's name and power limit.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

TOOLS = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--root", default=os.path.dirname(TOOLS))
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import k8s_spark_scheduler_b200 as g           # the package under test, imported before the workload modules
    sys.path.insert(0, TOOLS)
    import prepare_zones_bench as pz
    import prepare_zones_groups_bench as pzg

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    p = g.native.GangPacker()
    cases = []
    for n, Z in ((10000, 3), (50000, 8)):
        alloc, over, rnode, res, sort = pz.cluster(n + Z, n, Z, 100000)
        for kind in (g.native.LAYOUT_SINGLE_AZ, g.native.LAYOUT_AZ_AWARE):
            cases.append(("prepare_cluster_zones %d nodes %d zones %s" % (n, Z, "az-aware" if kind else "single-az"),
                          lambda alloc=alloc, over=over, rnode=rnode, res=res, sort=sort, kind=kind: p.prepare_cluster_zones(
                              alloc, over, rnode, res, sort["zone_id"], sort["n_zones"], sort["name_rank"], sort["is_driver_candidate"],
                              sort["unschedulable"], sort["ready"], sort["driver_label_rank"], None, kind=kind, layout=False)))
    if hasattr(p, "prepare_cluster_zones_groups"):
        alloc, over, rnode, res, sort, ig = pzg.cluster(10000, 16, 100000)
        for kind in (g.native.LAYOUT_SINGLE_AZ, g.native.LAYOUT_AZ_AWARE):
            cases.append(("prepare_cluster_zones_groups 10000 nodes 16 instance groups %s" % ("az-aware" if kind else "single-az"),
                          lambda kind=kind: p.prepare_cluster_zones_groups(alloc, over, rnode, res, ig, 16, *pzg.sort_args(sort),
                                                                           kind=kind, layout=False)))
    for name, call in cases:
        for _ in range(20):
            call()
        wall = []
        for _ in range(args.calls):
            t0 = time.perf_counter(); call(); wall.append(time.perf_counter() - t0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                call()
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            k = e.name.split("(")[0].replace("void ", "")
            c, us = per.get(k, (0, 0.0))
            per[k] = (c + 1, us + e.device_time)
        kernels = sorted(({"name": k, "per_call": c / args.calls, "us_per_call": round(us / args.calls, 2)} for k, (c, us) in per.items()),
                         key=lambda r: -r["us_per_call"])
        print(json.dumps({"root": root, "workload": name, "gpu": smi, "calls": args.calls,
                          "wall_ms_median": round(float(np.median(wall)) * 1e3, 3), "wall_ms_p10": round(float(np.percentile(wall, 10)) * 1e3, 3),
                          "device_us_per_call": round(sum(r["us_per_call"] for r in kernels), 2), "kernels": kernels}), flush=True)
    p.close()


if __name__ == "__main__":
    main()
