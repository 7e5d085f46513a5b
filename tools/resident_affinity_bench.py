"""Time the driver Predicate's affinity step from the resident label table against the per-call match it replaces.

    python tools/resident_affinity_bench.py [--reps 15] [--warmup 3] [--out FILE]

First, one profile of the per-call gp_match_node_affinity at 50 000 nodes x 20 labels (16 and 512 affinities) under
torch.profiler: device time of the label and program uploads (host-to-device copies), of gp_aff_labels and of gp_aff_match,
per call, next to the call's wall time -- how much of the per-call match is label staging.

Then clusters of N = 10 000 and 50 000 nodes with 20 and 60 labels each (tools/affinity_bench.py's generator: instance
group, zone, node type, cores, and "others" labels up to the count) and A = 1, 16 and 512 affinities from the same generator.
Each simulated Predicate first applies node events to an affinity.LabelTable: a churn of 0.1 % or 1 % of the nodes relabelled
(one "others" label changed, every tenth also its node type), two nodes deleted and two added.  Timed per Predicate:
  resident    LabelTable.flush (host delta + gp_label_table_update) + gp_match_node_affinity_resident, with the two parts
              also timed on their own (resident_update, resident_match)
  pinned      gp_match_node_affinity from page-locked label arrays (gp_alloc_pinned)
  pageable    gp_match_node_affinity from numpy label arrays
and the unschedulable-pod marker over 1 000 drivers: gp_exceeds_cluster_capacity_affinity_label_table against
gp_exceeds_cluster_capacity_affinity_resident on the same labels (an empty overhead table).  The per-call labels are the
table's mirror decoded (LabelTable.to_node_labels) and the programs LabelTable.encode_affinities, both made outside the timed
window: interning strings is the caller's on either side.  Every timed pair is checked to give the same answer.  Wall clock
(time.perf_counter) around each call, every one ending in a stream synchronise; medians with the 10th and 90th percentiles
over --reps Predicates after --warmup.  Prints the card's name and power limit, read in the same run.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import affinity as aff  # noqa: E402
from k8s_spark_scheduler_b200 import native  # noqa: E402
from affinity_bench import cluster  # noqa: E402

G = 1 << 30


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def stats(ts):
    ts = np.asarray(ts) * 1e3
    return {"median": round(float(np.median(ts)), 4), "p10": round(float(np.percentile(ts, 10)), 4),
            "p90": round(float(np.percentile(ts, 90)), 4)}


def nodes_with(rng, n, n_labels, n_aff):
    """affinity_bench.cluster's nodes with "others" labels added up to n_labels, and its affinities"""
    nodes, affs = cluster(rng, n, n_aff)
    for i, nd in enumerate(nodes):
        for j in range(16, n_labels - 4):
            nd["labels"][f"example.com/l{j}"] = f"v{(i * 7 + j) % 5}"
    return nodes, affs


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def profile_per_call(p, rng, reps=10):
    """device time per call of the uploads, gp_aff_labels and gp_aff_match inside gp_match_node_affinity"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    out = []
    for n_aff in (16, 512):
        nodes, affs = nodes_with(rng, 50_000, 20, n_aff)
        enc = aff.encode(nodes, affs)
        for _ in range(3):
            p.match_node_affinity(enc)
        wall = []
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                wall.append(timed(lambda: p.match_node_affinity(enc))[0])
        dev = {"h2d": 0.0, "d2h": 0.0, "memset": 0.0, "gp_aff_labels": 0.0, "gp_aff_match": 0.0, "other": 0.0}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            t = (e.time_range.end - e.time_range.start) / 1e3      # ms
            name = e.name
            key = ("h2d" if "HtoD" in name else "d2h" if "DtoH" in name else "memset" if "memset" in name.lower() else "gp_aff_labels" if "gp_aff_labels" in name else
                   "gp_aff_match" if "gp_aff_match" in name else "other")
            dev[key] += t
        label_bytes = sum(enc[k].nbytes for k in ("label_off", "label_key", "label_val", "label_int_ok", "label_int"))
        row = {"nodes": 50_000, "labels_per_node": 20, "affinities": n_aff, "calls": reps, "wall_ms": stats(wall),
               "device_ms_per_call": {k: round(v / reps, 4) for k, v in dev.items()}, "label_bytes": int(label_bytes)}
        print(json.dumps({"profile": row}), flush=True)
        out.append(row)
    return out


def churn(rng, t, live, serial, frac):
    for i in rng.choice(len(live), max(1, int(frac * len(live))), replace=False):
        name = live[i]
        lab = dict(t.labels[name])
        lab[f"example.com/l{int(rng.integers(0, 16))}"] = f"v{int(rng.integers(0, 9))}"
        if i % 10 == 0:
            lab["node-type"] = f"t{int(rng.integers(0, 4))}"
        t.set_node(name, lab)
    for _ in range(2):
        t.delete_node(live.pop(int(rng.integers(0, len(live)))))
    for _ in range(2):
        name = f"added-{serial[0]}"
        serial[0] += 1
        t.set_node(name, dict(t.labels[live[int(rng.integers(0, len(live)))]]))
        live.append(name)


def pinned_copy(p, enc, pool):
    """enc's label arrays copied into page-locked buffers (reused while large enough)"""
    out = dict(enc)
    for k in ("label_off", "label_key", "label_val", "label_int_ok", "label_int"):
        a = enc[k]
        buf = pool.get(k)
        if buf is None or buf.array.size < a.size:
            if buf is not None:
                buf.free()
            buf = native.PinnedArray(p, max(int(a.size * 1.2), 1), a.dtype)
            pool[k] = buf
        buf.array[:a.size] = a
        out[k] = buf.array[:a.size]
    return out


def run(p, rng, n, n_labels, n_aff, frac, reps, warmup):
    nodes, affs = nodes_with(rng, n, n_labels, n_aff)
    t = aff.LabelTable(n_node_ids=n, max_labels=n_labels, n_keys=256, n_values=1024)
    for nd in nodes:
        t.set_node(nd["name"], nd["labels"])
    t.flush(p)
    live, serial = [nd["name"] for nd in nodes], [0]
    q = 1000
    apps = {"drv_cpu": rng.integers(1, 5, q).astype(np.int64) * 1000, "drv_mem": rng.integers(1, 9, q).astype(np.int64) * G,
            "exe_cpu": rng.integers(1, 9, q).astype(np.int64) * 1000, "exe_mem": rng.integers(1, 33, q).astype(np.int64) * G,
            "count": rng.integers(1, 200, q).astype(np.int32), "group": rng.integers(0, n_aff, q).astype(np.int32)}
    pool = {}
    ts = {k: [] for k in ("resident", "resident_update", "resident_match", "pinned", "pageable", "marker_label_table",
                          "marker_affinity_resident")}
    update_rows = []
    try:
        for r in range(warmup + reps):
            churn(rng, t, live, serial, frac)
            rows_changed = len(t._dirty)
            t_res_flush, _ = timed(lambda: t.flush(p))
            ids = t.node_ids(live)
            progs = t.encode_affinities(affs, live)
            t_res_match, res = timed(lambda: p.match_node_affinity_resident(ids, progs))
            enc = dict(t.to_node_labels(ids), **progs)
            penc = pinned_copy(p, enc, pool)
            t_pin, pin = timed(lambda: p.match_node_affinity(penc))
            t_page, page = timed(lambda: p.match_node_affinity(enc))
            for a, b in ((res, pin), (res, page)):
                assert all(np.array_equal(x, y) for x, y in zip(a, b)), "resident and per-call matches differ"
            n_now = len(live)
            alloc = [np.full(n_now, 64_000, np.int64), np.full(n_now, 256 * G, np.int64), np.zeros(n_now, np.int64)]
            oids = np.full(n_now, -1, np.int32)
            t_mlt, m1 = timed(lambda: p.exceeds_cluster_capacity_affinity_label_table(alloc, oids, ids, progs, apps, 0))
            t_mar, m2 = timed(lambda: p.exceeds_cluster_capacity_affinity_resident(alloc, oids, enc, apps, 0))
            assert all(np.array_equal(x, y) for x, y in zip(m1, m2)), "marker entries differ"
            if r >= warmup:
                ts["resident"].append(t_res_flush + t_res_match)
                ts["resident_update"].append(t_res_flush)
                ts["resident_match"].append(t_res_match)
                ts["pinned"].append(t_pin)
                ts["pageable"].append(t_page)
                ts["marker_label_table"].append(t_mlt)
                ts["marker_affinity_resident"].append(t_mar)
                update_rows.append(rows_changed)
    finally:
        for b in pool.values():
            b.free()
    row = {"nodes": n, "labels_per_node": n_labels, "affinities": n_aff, "churn": frac, "rows_per_update": float(np.mean(update_rows)),
           "parity": True, **{k: stats(v) for k, v in ts.items()}}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    res = {"card": card()}
    print(json.dumps(res), flush=True)
    p = g.GangPacker()
    try:
        p.overhead_table_reset(1, 1, 1, 1, 1)
        res["profile_per_call"] = profile_per_call(p, rng)
        res["rows"] = [run(p, rng, n, L, A, frac, args.reps, args.warmup)
                       for n in (10_000, 50_000) for L in (20, 60) for A in (1, 16, 512) for frac in (0.001, 0.01)]
    finally:
        p.close()
    res["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
