#!/usr/bin/env python
"""Per-kernel device time of one bench.py step (snapshot layout + pack, device-resident inputs), from torch.profiler.
(diagnostic, not part of the bench contract)

    python tools/step_profile.py [--workload tightly-100k] [--steps 50] [--root TREE]

--root runs the package and bench.py workload of another checkout (e.g. the parent commit, built) for a before/after
table.  Prints one JSON line: the GPU's name and power limit, and per kernel its launches per step and mean µs per step."""
import argparse
import json
import os
import subprocess
import sys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="tightly-100k")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import k8s_spark_scheduler_b200 as g
    from bench import WORKLOADS, make_workload

    w = WORKLOADS[args.workload]
    nodes, a, eoff, eorder = make_workload(w, 0)
    dev = torch.device("cuda", 0)
    packer = g.GangPacker(device=0, async_snapshot=True)
    stream = torch.cuda.ExternalStream(packer.stream_handle(), device=dev)

    def t(x, dtype):
        return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).to(dev)

    tn = {"cpu": t(nodes["avail_cpu"], torch.int64), "mem": t(nodes["avail_mem"], torch.int64), "gpu": t(nodes["avail_gpu"], torch.int64),
          "eorder": t(eorder, torch.int32), "eoff": t(eoff, torch.int32)}
    keys = ["drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count"] + (["group"] if w["groups"] > 1 else [])
    ta = {k: t(a[k], torch.int64 if a[k].dtype == np.int64 else torch.int32) for k in keys}
    ta["off"] = t(a["off"], torch.int64)
    q = len(a["count"])
    d_driver = torch.empty(q, dtype=torch.int32, device=dev)
    d_exec = torch.empty(max(int(a["off"][-1]), 1), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()

    def step():
        packer.set_snapshot_device(tn["cpu"], tn["mem"], tn["gpu"], tn["eoff"], tn["eorder"], tn["eoff"], tn["eorder"])
        packer.pack_batch_device(ta, w["algo"], w["mode"], d_driver, d_exec)

    with torch.cuda.stream(stream):
        for _ in range(10):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        n, us = per.get(e.name, (0, 0.0))
        per[e.name] = (n + 1, us + e.device_time)
    kernels = sorted(({"name": k, "launches_per_step": n / args.steps, "us_per_step": us / args.steps} for k, (n, us) in per.items()),
                     key=lambda r: -r["us_per_step"])
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"root": root, "workload": args.workload, "gpu": smi, "steps": args.steps,
                      "sum_us_per_step": sum(r["us_per_step"] for r in kernels), "kernels": kernels}))
    torch.cuda.synchronize()
    packer.close()


if __name__ == "__main__":
    main()
