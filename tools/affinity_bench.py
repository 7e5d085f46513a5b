"""Time gp_match_node_affinity and gp_exceeds_cluster_capacity_affinity against the host recipes they replace.

    python tools/affinity_bench.py [--reps 10] [--warmup 2] [--out FILE]

Clusters: N = 10 000 and 50 000 nodes with 20 labels each (instance group of 32, zone of 8, node type of 4, 17 others) and
A = 16, 128 and 512 distinct required affinities built from them, so that most nodes match several affinities (instance-group
In lists, instance group + zone, node type NotIn, Gt on an integer label, a few nodeSelectors and name fields).
  match   one gp_match_node_affinity call  vs  the numpy evaluator of the same encoded programs (affinity.evaluate, host)
  marker  one gp_exceeds_cluster_capacity_affinity call over Q = 10 000 stale drivers spread over the affinities (tightly-pack)
          vs  today's recipe: host match (affinity.evaluate), then the affinities split greedily into groups with disjoint
          node sets and one gp_exceeds_cluster_capacity per group
Interning the strings is the same on both sides and is not timed.  Wall clock (time.perf_counter) around each complete
recipe, median of --reps after --warmup; every device call ends in a stream synchronise.  The answers of both sides are
checked to be equal.  Prints the card's name and power limit with the numbers.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import k8s_spark_scheduler_b200 as g  # noqa: E402
from k8s_spark_scheduler_b200 import affinity as aff  # noqa: E402

G = 1 << 30


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def cluster(rng, n, n_aff):
    ig, zone, typ = rng.integers(0, 32, n), rng.integers(0, 8, n), rng.integers(0, 4, n)
    nodes = []
    for i in range(n):
        lab = {"instance-group": f"ig{ig[i]}", "zone": f"z{zone[i]}", "node-type": f"t{typ[i]}", "cores": str(8 * (1 + i % 12))}
        lab.update({f"example.com/l{j}": f"v{(i * 7 + j) % 5}" for j in range(16)})
        nodes.append({"name": f"node-{i}", "labels": lab})
    affs = []
    for a in range(n_aff):
        r = a % 6
        if r == 0:
            t = [{"matchExpressions": [("instance-group", "In", [f"ig{x}" for x in rng.choice(32, 6, replace=False)])]}]
        elif r == 1:
            t = [{"matchExpressions": [("instance-group", "In", [f"ig{rng.integers(0, 32)}"]), ("zone", "In", [f"z{rng.integers(0, 8)}"])]}]
        elif r == 2:
            t = [{"matchExpressions": [("node-type", "NotIn", [f"t{rng.integers(0, 4)}"])]}]
        elif r == 3:
            t = [{"matchExpressions": [("cores", "Gt", [str(8 * int(rng.integers(1, 12)))])]},
                 {"matchExpressions": [("example.com/l3", "In", ["v1", "v2"])]}]
        elif r == 4:
            t = [{"matchExpressions": [("zone", "In", ["z0", "z1", "z2", "z3"])],
                  "matchFields": [("metadata.name", "NotIn", [f"node-{rng.integers(0, n)}"])]}]
        else:
            t = None
        affs.append({"nodeSelector": {"example.com/l0": f"v{a % 5}"} if r == 5 else None, "required": t})
    return nodes, affs


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, out


def disjoint_groups(sets, n):
    """greedy: each affinity goes to the first group none of whose nodes it matches"""
    groups, used = [], []
    for a, m in enumerate(sets):
        for gi, u in enumerate(used):
            if not u[m].any():
                groups[gi].append(a); u[m] = True
                break
        else:
            u = np.zeros(n, bool); u[m] = True
            groups.append([a]); used.append(u)
    return groups


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    p = g.GangPacker()
    rows = []
    try:
        for n in (10_000, 50_000):
            alloc = [rng.integers(8, 97, n).astype(np.int64) * 1000, rng.integers(32, 385, n).astype(np.int64) * G, np.zeros(n, np.int64)]
            for n_aff in (16, 128, 512):
                nodes, affs = cluster(rng, n, n_aff)
                enc = aff.encode(nodes, affs)
                t_dev, (member, _, _) = timed(lambda: p.match_node_affinity(enc), args.reps, args.warmup)
                t_host, (outcome, h_member, _, _) = timed(lambda: aff.evaluate(enc), max(1, args.reps // 5), 0)
                assert np.array_equal(member, h_member)
                q = 10_000
                apps = {"drv_cpu": rng.integers(1, 5, q).astype(np.int64) * 1000, "drv_mem": rng.integers(1, 9, q).astype(np.int64) * G,
                        "exe_cpu": rng.integers(1, 9, q).astype(np.int64) * 1000, "exe_mem": rng.integers(1, 33, q).astype(np.int64) * G,
                        "count": rng.integers(1, 2000, q).astype(np.int32), "group": rng.integers(0, n_aff, q).astype(np.int32)}
                t_new, (ex_new, _) = timed(lambda: p.exceeds_cluster_capacity_affinity(alloc, enc, apps, 0), args.reps, args.warmup)

                def old():
                    sets = [np.nonzero(r == 1)[0] for r in aff.evaluate(enc)[0]]
                    out = np.zeros(q, np.uint8)
                    groups = disjoint_groups(sets, n)
                    for grp in groups:
                        cls = np.full(n, -1, np.int32)
                        for k, a in enumerate(grp):
                            cls[sets[a]] = k
                        local = np.full(n_aff, -1, np.int64); local[grp] = np.arange(len(grp))
                        idx = np.nonzero(local[apps["group"]] >= 0)[0]
                        part = {k: v[idx] for k, v in apps.items()}
                        part["group"] = local[part["group"]].astype(np.int32)
                        out[idx] = p.exceeds_cluster_capacity(alloc, part, 0, node_group=cls, n_groups=len(grp))
                    return out, len(groups)

                t_old, (ex_old, n_calls) = timed(old, max(1, args.reps // 5), 0)
                assert np.array_equal(ex_new, ex_old)
                row = dict(nodes=n, affinities=n_aff, memberships_per_node=float((outcome == 1).sum(0).mean()),
                           match_device_ms=round(t_dev, 3), match_host_numpy_ms=round(t_host, 3),
                           marker_device_ms=round(t_new, 3), marker_host_match_plus_disjoint_calls_ms=round(t_old, 3),
                           disjoint_calls=n_calls)
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
