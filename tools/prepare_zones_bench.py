"""Time gp_prepare_cluster_zones against the host recipe it replaces, for the zone-aware packers' snapshot.

    python tools/prepare_zones_bench.py [--reps 30] [--warmup 5] [--kind az-aware|single-az] [--out FILE]

Per (nodes, zones) point, 100 000 reservations: one prepare_cluster_zones call (reservations -> availability -> orders ->
zone-grouped snapshot + SchedulableResources, one synchronise) against gp_build_availability -> gp_potential_nodes -> grouping
in numpy -> gp_set_snapshot -> gp_set_schedulable.  Both are timed with a wall clock around calls that end in a stream
synchronise, alternating, after warm-up; the script checks that both leave the same layout and prints median and best with
the card's name and power limit.  Needs a GPU."""
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
    alloc = [rng.integers(8, 97, n) * 1000, rng.integers(32, 385, n) * G, np.zeros(n, np.int64)]
    over = [rng.integers(0, 3, n) * 250, rng.integers(0, 4, n) * (1 << 28), np.zeros(n, np.int64)]
    rnode = rng.integers(-1, n, R).astype(np.int32)
    res = [rng.integers(0, 6, R) * 500, rng.integers(0, 12, R) * (1 << 29), np.zeros(R, np.int64)]
    zid = rng.integers(0, Z, n).astype(np.int32)
    seen = {}
    zid = np.array([seen.setdefault(int(z), len(seen)) for z in zid], np.int32)
    names = np.argsort(rng.permutation(n)).astype(np.int32)
    sort = dict(zone_id=zid, n_zones=len(seen), name_rank=names, is_driver_candidate=(rng.random(n) < 0.8).astype(np.uint8),
                unschedulable=(rng.random(n) < 0.05).astype(np.uint8), ready=(rng.random(n) < 0.95).astype(np.uint8),
                driver_label_rank=rng.integers(-1, 3, n).astype(np.int32))
    return alloc, over, rnode, res, sort


def numpy_grouping(d, e, zid, kind):
    """binpack::ZoneGroups / AzAwareLayout over index arrays -> (exec_order, drv_order, exec_off, drv_off, n_zones)"""
    dz, ez = zid[d], zid[e]
    zones, first = np.unique(dz, return_index=True)
    keep = np.isin(zones, ez)
    cand = zones[keep][np.argsort(first[keep], kind="stable")]
    nz = len(cand)
    zone_group = np.full(int(zid.max()) + 1 if len(zid) else 1, -1, np.int64)
    zone_group[cand] = np.arange(nz)
    rest = nz if kind == g.native.LAYOUT_AZ_AWARE else -1
    out, trailing = [], False
    for order, oz in ((e, ez), (d, dz)):
        r = zone_group[oz]
        trailing |= bool((r < 0).any())
        r = np.where(r < 0, rest, r)
        key = np.where(r < 0, np.iinfo(np.int64).max, r)
        perm = np.argsort(key, kind="stable")
        out.append((order[perm], key[perm]))
    if kind == g.native.LAYOUT_AZ_AWARE:
        n_groups = nz + (1 if (trailing or nz == 0) else 0)
    else:
        n_groups = max(nz, 1)
    offs = [np.searchsorted(k, np.arange(n_groups + 1), side="left").astype(np.int32) for _, k in out]
    return out[0][0][:offs[0][-1]].astype(np.int32), out[1][0][:offs[1][-1]].astype(np.int32), offs[0], offs[1], nz


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
    ap.add_argument("--kind", choices=("az-aware", "single-az"), default="az-aware")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    kind = g.native.LAYOUT_AZ_AWARE if a.kind == "az-aware" else g.native.LAYOUT_SINGLE_AZ
    dev, host = g.native.GangPacker(), g.native.GangPacker()
    print(json.dumps({"card": card(), "kind": a.kind, "reps": a.reps}), flush=True)
    lines = []
    for n in (10000, 50000):
        for Z in (3, 8, 16):
            alloc, over, rnode, res, sort = cluster(n + Z, n, Z, 100000)

            def device():
                return dev.prepare_cluster_zones(alloc, over, rnode, res, sort["zone_id"], sort["n_zones"], sort["name_rank"],
                                                 sort["is_driver_candidate"], sort["unschedulable"], sort["ready"],
                                                 sort["driver_label_rank"], None, kind=kind, layout=False)

            def recipe():
                av, sc = host.build_availability(alloc, over, rnode, res)
                d, e = host.potential_nodes(av[0], av[1], sort["zone_id"], sort["n_zones"], sort["name_rank"], sort["is_driver_candidate"],
                                            sort["unschedulable"], sort["ready"], sort["driver_label_rank"], None)
                eo, do, eoff, doff, nz = numpy_grouping(d, e, sort["zone_id"], kind)
                host.set_snapshot(av[0], av[1], av[2], eo, do, eoff, doff)
                host.set_schedulable(*sc)
                return eo, do, eoff, doff, nz

            full = dev.prepare_cluster_zones(alloc, over, rnode, res, sort["zone_id"], sort["n_zones"], sort["name_rank"],
                                             sort["is_driver_candidate"], sort["unschedulable"], sort["ready"],
                                             sort["driver_label_rank"], None, kind=kind)
            eo, do, eoff, doff, nz = recipe()
            assert full["n_zones"] == nz and np.array_equal(full["exec_off"], eoff) and np.array_equal(full["drv_off"], doff)
            assert np.array_equal(full["exec_order"], eo) and np.array_equal(full["drv_order"], do)
            for x, y in zip(dev.get_snapshot(), host.get_snapshot()):
                assert np.array_equal(x, y)
            for _ in range(a.warmup):
                device(); recipe()
            td, th = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter(); device(); td.append(time.perf_counter() - t0)
                t0 = time.perf_counter(); recipe(); th.append(time.perf_counter() - t0)
            r = dict(nodes=n, zones=Z, reservations=100000, candidate_zones=nz,
                     device_ms_median=round(1e3 * float(np.median(td)), 3), device_ms_best=round(1e3 * min(td), 3),
                     host_recipe_ms_median=round(1e3 * float(np.median(th)), 3), host_recipe_ms_best=round(1e3 * min(th), 3))
            r["speedup_median"] = round(r["host_recipe_ms_median"] / r["device_ms_median"], 2)
            print(json.dumps(r), flush=True)
            lines.append(r)
    dev.close(); host.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "kind": a.kind, "results": lines}, f, indent=1)


if __name__ == "__main__":
    main()
