"""Time gp_placement_metrics -- the Predicate's collocation, executor node count and cross-zone pod pairs -- on the
tightly-100k batch (10 000 nodes x 100 000 applications, tightly-pack, independent), next to the host restatements.

    python tools/placement_metrics_bench.py [--reps 30] [--warmup 5] [--out FILE]

Paths, all on the same placement and metric-zone column (6 failure-domain zones, every 11th node unlabelled, so it lands
in "unknown-zone"):
  host form     GangPacker.placement_metrics on host arrays: upload, kernels, download, one synchronise (host clock)
  device form   gp_placement_metrics_device on the outputs of gp_pack_batch_device, in place (CUDA events on the stream)
  literal       tests/placement_metrics_ref.literal_batch: the string-keyed restatement of the three reporters (one run)
  numpy         tests/placement_metrics_ref.closed_form: the closed form per row in numpy (one run)
Every path must give the same records.  Prints the card's name, power limit and SM clock with the numbers, and writes them
as JSON to tools/results/placement_metrics_bench_h100.json (or --out).  Needs a GPU: without one it fails and writes
nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import synth  # noqa: E402
import placement_metrics_ref as ref  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "results", "placement_metrics_bench_h100.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("placement_metrics_bench: no GPU; nothing measured")
    n, q = 10000, 100000
    nodes = synth.make_nodes(n)
    apps = synth.make_apps(q)
    off = synth.exec_offsets(apps["count"])
    eoff, eorder = synth.group_orders(nodes)
    labels = [{} if v % 11 == 0 else {ref.LABEL_ZONE_FAILURE_DOMAIN: "zone-%d" % (v % 6)} for v in range(n)]
    zone, nz = ref.intern_metric_zones(labels)
    names = synth.node_names(n)

    p = g.GangPacker()
    try:
        p.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
        dev = torch.device("cuda", 0)
        t = {k: torch.from_numpy(np.ascontiguousarray(apps[k])).to(dev) for k in ("drv_cpu", "drv_mem", "exe_cpu", "exe_mem", "count")}
        t["off"] = torch.from_numpy(off).to(dev)
        d_drv = torch.empty(q, dtype=torch.int32, device=dev)
        d_exe = torch.empty(int(off[-1]), dtype=torch.int32, device=dev)
        p.pack_batch_device(t, g.TIGHTLY_PACK, g.MODE_INDEPENDENT, d_drv, d_exe)
        p.synchronize()
        placed = (d_drv.cpu().numpy(), d_exe.cpu().numpy(), off)
        host_apps = {"count": apps["count"], "off": off}

        # host form
        for _ in range(args.warmup):
            p.placement_metrics(host_apps, placed, zone)
        host_ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rec = p.placement_metrics(host_apps, placed, zone)
            host_ms.append((time.perf_counter() - t0) * 1e3)

        # device form, reading gp_pack_batch_device's outputs in place
        d_zone = torch.from_numpy(zone).to(dev)
        out = torch.empty(g.native.PLACEMENT_DTYPE.itemsize * q, dtype=torch.uint8, device=dev)
        status = torch.empty(1, dtype=torch.int32, device=dev)
        stream = torch.cuda.ExternalStream(p.stream_handle())
        for _ in range(args.warmup):
            p.placement_metrics_device(t, d_drv, d_exe, d_zone, out, nz, status=status)
        dev_ms = []
        for _ in range(args.reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(stream)
            p.placement_metrics_device(t, d_drv, d_exe, d_zone, out, nz, status=status)
            e.record(stream)
            e.synchronize()
            dev_ms.append(s.elapsed_time(e))
        p.synchronize()
        assert int(status.item()) == 0
        dev_rec = out.cpu().numpy().view(g.native.PLACEMENT_DTYPE)
    finally:
        p.close()

    t0 = time.perf_counter()
    lit = np.asarray(ref.literal_batch(*placed, apps["count"], names, labels, rng=np.random.default_rng(1)), np.int64)
    literal_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    cf = ref.closed_form(*placed, apps["count"], zone)
    numpy_ms = (time.perf_counter() - t0) * 1e3
    rows = ref.records_to_rows(rec)
    same = bool(np.array_equal(rows, lit) and np.array_equal(rows, cf) and dev_rec.tobytes() == rec.tobytes())

    med = lambda x: float(np.median(x))  # noqa: E731
    res = {"card": card(), "workload": "tightly-100k placement (10 000 nodes, 100 000 applications)",
           "placed_rows": int((placed[0] >= 0).sum()), "executor_entries": int(off[-1]), "n_metric_zones": nz,
           "host_form_ms": {"median": med(host_ms), "min": min(host_ms), "max": max(host_ms)},
           "device_form_ms": {"median": med(dev_ms), "min": min(dev_ms), "max": max(dev_ms)},
           "literal_ms": literal_ms, "numpy_ms": numpy_ms, "reps": args.reps, "all_paths_equal": same}
    print(json.dumps(res), flush=True)
    if not same:
        raise SystemExit("placement_metrics_bench: the paths disagree")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
