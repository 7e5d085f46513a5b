"""Time gp_packing_efficiency -- the Predicate's cluster-wide packing efficiency, exactly summed -- on the device, next to the
host time of the literal oracle's ComputePackingEfficiencies + ComputeAvgPackingEfficiency.

    python tools/efficiency_bench.py [--reps 30] [--warmup 5] [--out FILE]

Points: (N = 10 000, Q = 1), (N = 50 000, Q = 1), (N = 10 000, Q = 100 000) placed tightly-pack rows.  Device time: CUDA
events recorded on the context's stream around each call (base pass, partial reduction and row pass; the call's H2D of the
placement and D2H of the averages are inside the window).  Host time: orc_binpack with with_efficiencies = 1 minus the same
call without, for one application, on the same cluster and placement, difference of the medians (the O(N) metrics pass the reference runs after every
successful pack).  Prints the card's name and power limit with the numbers.  Needs a GPU."""
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


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def cluster(rng, n):
    sc = rng.integers(8, 97, n) * 1000 + rng.integers(0, 2, n) * 500
    sm = rng.integers(32, 385, n) * G
    sg = (rng.integers(0, 8, n) == 0) * 4
    avail = [sc - rng.integers(0, 8, n) * 1000, sm - rng.integers(0, 32, n) * G, sg - (sg > 0) * rng.integers(0, 3, n)]
    return [np.asarray(x, np.int64) for x in avail], [np.asarray(x, np.int64) for x in (sc, sm, sg)]


def apps_of(rng, q):
    """q applications; a single one always has 16 executors of 2 cores / 4 GiB, so the one-row points differ in N only"""
    if q == 1:
        return {"drv_cpu": np.full(1, 1000, np.int64), "drv_mem": np.full(1, 2 * G, np.int64), "drv_gpu": np.zeros(1, np.int64),
                "exe_cpu": np.full(1, 2000, np.int64), "exe_mem": np.full(1, 4 * G, np.int64), "exe_gpu": np.zeros(1, np.int64),
                "count": np.full(1, 16, np.int32)}
    return {"drv_cpu": np.full(q, 1000, np.int64), "drv_mem": np.full(q, 2 * G, np.int64), "drv_gpu": np.zeros(q, np.int64),
            "exe_cpu": rng.integers(1, 5, q).astype(np.int64) * 1000, "exe_mem": rng.integers(1, 9, q).astype(np.int64) * G,
            "exe_gpu": np.zeros(q, np.int64), "count": rng.integers(1, 33, q).astype(np.int32)}


def device_ms(p, apps, placed, reps, warmup):
    import torch
    stream = torch.cuda.ExternalStream(p.stream_handle())
    for _ in range(warmup):
        p.packing_efficiency(apps, placed, g.TIGHTLY_PACK)
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(stream)
        p.packing_efficiency(apps, placed, g.TIGHTLY_PACK)
        e.record(stream)
        e.synchronize()
        times.append(s.elapsed_time(e))
    return times


def host_ms(avail, sched, apps, order_names, reps):
    from oracle import oracle as orc
    orc.build()
    n = len(avail[0])
    names = ["node-%06d" % i for i in range(n)]
    cl = orc.Cluster(names, *avail, sched=sched)
    dr = (int(apps["drv_cpu"][0]), int(apps["drv_mem"][0]), int(apps["drv_gpu"][0]))
    er = (int(apps["exe_cpu"][0]), int(apps["exe_mem"][0]), int(apps["exe_gpu"][0]))
    k = int(apps["count"][0])
    on = [names[i] for i in order_names]

    def once(eff):
        t0 = time.perf_counter()
        cl.binpack(0, dr, er, k, on, on, with_efficiencies=eff)
        return (time.perf_counter() - t0) * 1e3
    once(True); once(False)                      # warm-up
    with_eff, without = [], []
    for _ in range(3 * reps):                    # alternate the two so that drift hits both
        with_eff.append(once(True))
        without.append(once(False))
    return with_eff, without


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    rows = []
    p = g.GangPacker()
    try:
        for n, q in ((10_000, 1), (50_000, 1), (10_000, 100_000)):
            rng = np.random.default_rng(n + q)
            avail, sched = cluster(rng, n)
            order = rng.permutation(n).astype(np.int32)
            p.set_snapshot(*avail, order, order)
            p.set_schedulable(*sched)
            apps = apps_of(rng, q)
            placed = p.pack_batch(apps, g.TIGHTLY_PACK)
            dev = device_ms(p, apps, placed, args.reps, args.warmup)
            row = {"nodes": n, "rows": q, "placed": int((placed[0] >= 0).sum()),
                   "device_ms_median": float(np.median(dev)), "device_ms_best": float(np.min(dev))}
            if q == 1:
                with_eff, without = host_ms(avail, sched, apps, order, args.reps)
                row.update(host_pack_with_efficiencies_ms_median=float(np.median(with_eff)),
                           host_pack_without_ms_median=float(np.median(without)),
                           host_metrics_ms_median=float(np.median(with_eff) - np.median(without)))
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
