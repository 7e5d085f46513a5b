"""Time gp_reschedule_from_reservations against the five-call sequence it replaces, for one executor Predicate.

    python tools/reschedule_bench.py [--reps 30] [--warmup 5] [--execs 1] [--out FILE]

Per (nodes, zones, branch, label ranking) point, 100 000 reservation rows: one reschedule_from_reservations call
(reservations -> both availabilities -> arg-min decision, one synchronise) against gp_build_availability ->
gp_build_reschedule_availability -> gp_potential_nodes -> gp_set_snapshot -> gp_reschedule_executors on a second context.
Both are timed with a wall clock around calls that end in a stream synchronise, alternating, after warm-up; the script
checks that both choose the same nodes and prints median and best with the card's name and power limit.  Needs a GPU."""
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


def cluster(seed, n, Z, R):
    rng = np.random.default_rng(seed)
    alloc = [rng.integers(8, 97, n) * 1000, rng.integers(32, 385, n) * G, (rng.integers(0, 8, n) == 0) * 4]
    over = [rng.integers(0, 3, n) * 250, rng.integers(0, 4, n) * (1 << 28), np.zeros(n, np.int64)]
    rnode = rng.integers(-1, n, R).astype(np.int32)
    res = [rng.integers(0, 6, R) * 500, rng.integers(0, 12, R) * (1 << 29), np.zeros(R, np.int64)]
    zid = rng.integers(0, Z, n).astype(np.int32)
    seen = {}
    zid = np.array([seen.setdefault(int(z), len(seen)) for z in zid], np.int32)
    names = np.argsort(rng.permutation(n)).astype(np.int32)
    sort = dict(zone_id=zid, n_zones=len(seen), name_rank=names, unschedulable=(rng.random(n) < 0.05).astype(np.uint8),
                ready=(rng.random(n) < 0.95).astype(np.uint8), executor_label_rank=rng.integers(-1, 3, n).astype(np.int32))
    return alloc, over, rnode, res, sort


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except Exception as ex:          # the numbers are still printed; the card line says why it is missing
        return f"unknown ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--execs", type=int, default=1, help="executors decided per call")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev, host = g.native.GangPacker(), g.native.GangPacker()
    print(json.dumps({"card": card(), "reps": a.reps, "execs": a.execs}), flush=True)
    lines = []
    for n in (10000, 50000):
        for Z in (3, 16):
            alloc, over, rnode, res, sort = cluster(n + Z, n, Z, 100000)
            rng = np.random.default_rng(n * Z)
            exe = (rng.integers(1, 9, a.execs) * 500, rng.integers(1, 17, a.execs) * (G // 2), np.zeros(a.execs, np.int64))
            hosting = [list(rng.integers(0, n, 4)) for _ in range(a.execs)]
            for mf in (False, True):
                for labels in (False, True):
                    lre = sort["executor_label_rank"] if labels else None

                    def device():
                        return dev.reschedule_from_reservations(alloc, over, rnode, res, exe, min_frag=mf, hosting=hosting,
                                                                zone_id=sort["zone_id"], n_zones=sort["n_zones"],
                                                                name_rank=sort["name_rank"], unschedulable=sort["unschedulable"],
                                                                ready=sort["ready"], executor_label_rank=lre)[0]

                    def recipe():
                        meta, _ = host.build_availability(alloc, over, rnode, res)
                        ff = host.build_reschedule_availability(alloc, over, rnode, res)
                        _, eo = host.potential_nodes(meta[0], meta[1], sort["zone_id"], sort["n_zones"], sort["name_rank"], None,
                                                     sort["unschedulable"], sort["ready"], None, lre)
                        av = meta if mf else ff
                        host.set_snapshot(av[0], av[1], av[2], eo, eo)
                        return host.reschedule_executors(exe, min_frag=mf, reserved=over if mf else None, hosting=hosting if mf else None)

                    assert np.array_equal(device(), recipe()), (n, Z, mf, labels)
                    for _ in range(a.warmup):
                        device(); recipe()
                    td, th = [], []
                    for _ in range(a.reps):
                        t0 = time.perf_counter(); device(); td.append(time.perf_counter() - t0)
                        t0 = time.perf_counter(); recipe(); th.append(time.perf_counter() - t0)
                    r = dict(nodes=n, zones=Z, reservations=100000, branch="min-frag" if mf else "first-fit", label_rank=labels,
                             device_ms_median=round(1e3 * float(np.median(td)), 3), device_ms_best=round(1e3 * min(td), 3),
                             five_calls_ms_median=round(1e3 * float(np.median(th)), 3), five_calls_ms_best=round(1e3 * min(th), 3))
                    r["speedup_median"] = round(r["five_calls_ms_median"] / r["device_ms_median"], 2)
                    print(json.dumps(r), flush=True)
                    lines.append(r)
    dev.close(); host.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "execs": a.execs, "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
