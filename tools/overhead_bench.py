"""Time gp_node_overhead against a string-keyed restatement of the overhead computer it replaces.

    python tools/overhead_bench.py [--reps 10] [--warmup 3] [--out FILE]

Clusters (overhead.synthetic_cluster, seeded): 10 000 nodes x 300 000 pod records and 50 000 x 1 000 000, each with ~3
non-spark pods per node, a tail of large applications (20 and 40 of 2 000 executors) and small ones (0-40 executors) across
16 namespaces; most applications hold a ResourceReservation, some soft reservations; 1 % of the records are absent from the
lister.  Every node is listed, as one call for a whole marker scan would.
  device       one gp_node_overhead call, wall clock around it (it ends in a stream synchronise), median of --reps after
               --warmup, with the inputs in ordinary (pageable) numpy arrays and again in page-locked ones (GangPacker.pinned)
  split        one further call of each kind under torch.profiler (CUDA activities): the device time of the host-to-device
               copies, of the kernels and of the device-to-host copies, as the trace lists them
  bytes        host-to-device and device-to-host bytes of the call, computed from the shapes
  restatement  tests/overhead_ref.py's getOverheadByNode over the same strings, single-threaded Python on the same host --
               a restatement, not Go; its per-node answers and the numpy evaluator's are checked equal to the device's
Interning the strings is not timed.  Prints the card's name and power limit, read in the same run.  Needs a GPU."""
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
from k8s_spark_scheduler_b200 import overhead as oh  # noqa: E402
import overhead_ref as ref  # noqa: E402

ARRAYS = ("node_id", "req_cpu_milli", "req_mem_bytes", "req_gpu", "listed", "app_key", "app_id", "name_id", "is_executor",
          "spark_scheduler", "rr_app_key", "rr_pod_off", "rr_pod_name", "soft_app_id", "soft_pod_off", "soft_pod_name", "node_ids")


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, out


def split(fn):
    """-> (H2D ms, kernel ms, D2H ms) of one call, from a torch.profiler trace"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    h2d = ker = d2h = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if "HtoD" in e.key:
            h2d += t
        elif "DtoH" in e.key:
            d2h += t
        elif e.key.startswith("gp_oh_") or "gp::gp_oh_" in e.key:
            ker += t
    return round(h2d / 1e3, 3), round(ker / 1e3, 3), round(d2h / 1e3, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    p = g.GangPacker()
    rows = []
    try:
        for seed, (n, q, big) in enumerate([(10_000, 300_000, 20), (50_000, 1_000_000, 40)]):
            nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(seed, n, q, big_apps=big, big_executors=2000)
            enc = oh.encode(rec.slots, lister, rrs, soft, nodes)
            t_dev, (ov, ns, has, warned) = timed(lambda: p.node_overhead(enc), args.reps, args.warmup)
            pinned = dict(enc)
            for k in ARRAYS:
                pinned[k] = p.pinned(enc[k].shape, enc[k].dtype)
                pinned[k][...] = enc[k]
            t_pin, (ov2, ns2, has2, warned2) = timed(lambda: p.node_overhead(pinned), args.reps, args.warmup)
            split_pageable, split_pinned = split(lambda: p.node_overhead(enc)), split(lambda: p.node_overhead(pinned))
            e_ov, e_ns, e_has, e_warned = oh.evaluate(enc)

            def restate():
                comp = ref.OverheadComputer()
                for pod in pods:
                    comp.on_add(pod)
                t0 = time.perf_counter()
                ov_r, ns_r, w_r = comp.get_overhead_by_node(nodes, lister, rrs, soft)
                return time.perf_counter() - t0, (ref.columns(nodes, ov_r), ref.columns(nodes, ns_r), w_r)

            t_ref, want = restate()
            got = (tuple(list(map(int, c)) for c in ov), tuple(list(map(int, c)) for c in ns), warned)
            agree = (tuple(got[0]), tuple(got[1]), got[2]) == want
            agree &= all(np.array_equal(a, b) for a, b in zip(ov + ns, e_ov + e_ns)) and np.array_equal(has, e_has) and warned == e_warned
            agree &= all(np.array_equal(a, b) for a, b in zip(ov + ns, ov2 + ns2)) and np.array_equal(has, has2) and warned == warned2
            assert agree, "device, evaluator and restatement disagree"
            up = sum(enc[k].nbytes for k in ARRAYS)
            down = 48 * n + q + 16
            row = dict(nodes=n, pod_records=q, reserved_entries=int(enc["rr_pod_off"][-1] + enc["soft_pod_off"][-1]),
                       has_reservation=int(has.sum()), warned=warned,
                       device_call_ms_pageable=round(t_dev, 3), device_call_ms_pinned=round(t_pin, 3),
                       split_ms_pageable_h2d_kernels_d2h=split_pageable, split_ms_pinned_h2d_kernels_d2h=split_pinned,
                       h2d_bytes=up, h2d_bytes_per_pod_record=round(up / q, 2), d2h_bytes=down,
                       restatement_not_go_ms=round(t_ref * 1e3, 1), agrees_with_restatement=bool(agree))
            rows.append(row)
            print(json.dumps(row), flush=True)
    finally:
        p.close()
    res = {"card": card(), "rows": rows}
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
