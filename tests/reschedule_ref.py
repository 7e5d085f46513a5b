"""rescheduleExecutor (EXT/resource.go:594-673) restated literally for the tests of gp_reschedule_from_reservations, plus the
numpy arg-min formulation the device implements (DESIGN.md §2).

EXT = /root/reference/internal/extender.  Resources are (cpu_milli, mem_bytes, gpu) tuples; nodes are addressed by name in
the literal part (dicts, like the reference) and by index in the model.  Test infrastructure only: small cases.
"""
from __future__ import annotations

import itertools

import numpy as np

from oracle import pyref

ZONE_LABEL = "topology.kubernetes.io/zone"      # v1.LabelTopologyZone


class ReferenceError(Exception):
    """An error the reference returns (werror.ErrorWithContextParams)."""


def filter_nodes_to_zone(initial_nodes, node_labels, zone):
    """filterNodesToZone, EXT/resource.go:463-478: the nodes whose zone label equals `zone`, in order; ANY node without the
    label -- of this zone or another -- fails the whole call (:467-469)."""
    nodes = []
    for node in initial_nodes:
        labels = node_labels[node]
        if ZONE_LABEL not in labels:
            raise ReferenceError("Could not read zone label from node, unable to make scheduling decisions based on AZ")
        if labels[ZONE_LABEL] == zone:
            nodes.append(node)
    return nodes


def get_common_zone_for_executors_application(executor_labels, application_pods, node_labels):
    """getCommonZoneForExecutorsApplication, EXT/resource.go:493-516, with filterToRunningPods (:536-545) and getAzsOfPods
    (:518-533).  application_pods: [(phase, node_name)] of the application's pods (getSparkApplicationPodsForExecutor);
    node_labels: node name -> labels (a missing name is the lister's error).  -> (zone, True) when every running pod sits in
    one zone, ("", False) when they span several; raises ReferenceError otherwise."""
    if "spark-app-id" not in executor_labels:                                         # :494-497 (common.SparkAppIDLabel)
        raise ReferenceError("Executor does not have a Spark app id label, could not create label selector")
    scheduled = [(phase, node) for phase, node in application_pods if phase == "Running"]   # filterToRunningPods
    azs = set()
    for _, node in scheduled:                                                         # getAzsOfPods :520-531
        if node not in node_labels:
            raise ReferenceError("node %s not found" % node)
        labels = node_labels[node]
        if ZONE_LABEL not in labels:
            raise ReferenceError("Could not read zone label from node, unable to make scheduling decisions based on AZ")
        azs.add(labels[ZONE_LABEL])
    if len(azs) > 1:                                                                  # :508-510
        return "", False
    if len(azs) == 0:                                                                 # :511-513
        raise ReferenceError("Application has no scheduled pods, can't make scheduling decisions based on AZ")
    return next(iter(azs)), True


def first_fit_available(alloc, overhead, reservations):
    """availableResources of rescheduleExecutor (:638-643): NodeSchedulingMetadataForNodes adds the overhead into the usage
    map's EXISTING entries in place (LIB/resources/resources.go:72-76), then usage.Add(overhead) adds it once more (App. B7)."""
    usage = {}
    for node, r in reservations:
        usage[node] = pyref.add(usage.get(node, pyref.ZERO), r)
    for n in alloc:                                   # NodeSchedulingMetadataForNodes, in place on existing entries
        if n in usage:
            usage[n] = pyref.add(usage[n], overhead.get(n, pyref.ZERO))
    for n, o in overhead.items():                     # usage.Add(overhead)
        usage[n] = pyref.add(usage.get(n, pyref.ZERO), o)
    return {n: pyref.sub(a, usage.get(n, pyref.ZERO)) for n, a in alloc.items()}


def reschedule_executor(nodes, node_labels, sort_zone, alloc, overhead, reservations, unschedulable, not_ready, exec_label_rank,
                        exe, min_frag, hosting, common_zone=None):
    """rescheduleExecutor's node choice (:594-673) without pod / lister I/O.  nodes: availableNodes in table order; sort_zone:
    name -> ZoneLabel as the sorter sees it; common_zone: the zone getCommonZoneForExecutorsApplication returned, or None.
    -> the node name, or None (failureFit)."""
    exec_order, meta, ff, ov = executor_state(nodes, node_labels, sort_zone, alloc, overhead, reservations, unschedulable,
                                              not_ready, exec_label_rank, common_zone)
    return choose(exe, min_frag, hosting, exec_order, meta, ff, ov)


def executor_state(nodes, node_labels, sort_zone, alloc, overhead, reservations, unschedulable, not_ready, exec_label_rank,
                   common_zone=None):
    """:604-642 -> (executorNodeNames, availableNodesSchedulingMetadata, availableResources, overhead)."""
    available = list(nodes)
    if common_zone is not None:
        available = filter_nodes_to_zone(available, node_labels, common_zone)            # :621
    al = {n: alloc[n] for n in available}
    ov = {n: overhead.get(n, pyref.ZERO) for n in available}                              # GetOverhead(availableNodes) :636
    meta, _ = pyref.node_scheduling_metadata(al, ov, reservations)                         # :637
    ff = first_fit_available(al, ov, reservations)                                         # :639-640
    _, exec_order = pyref.potential_nodes(meta, sort_zone, [], unschedulable=unschedulable, not_ready=not_ready,
                                          exec_label_rank=exec_label_rank)                 # :642
    return exec_order, meta, ff, ov


def choose(exe, min_frag, hosting, exec_order, meta, ff, ov):
    """:649-662: the one decision over executorNodeNames."""
    if min_frag:
        return pyref.reschedule_minimal_fragmentation(exe, exec_order, meta, ov, hosting)
    return pyref.reschedule_first_fit(exe, exec_order, ff)


# ---- the arg-min formulation (what gangpack_reschedprep.cuh computes) ----------------------------------------------------
def capacity(v, e):
    """GetNodeCapacities' per-node minimum over dimensions of (v >= 0 ? (e ? v // e : MaxInt) : 0), v = avail - reserved."""
    c = pyref.MAX_INT
    for d in range(3):
        c = min(c, 0 if v[d] < 0 else (pyref.MAX_INT if e[d] == 0 else v[d] // e[d]))
    return c


def zone_priority(meta, zone, member):
    """rank of each zone id by (Σ mem, Σ cpu, id) over the member nodes (nodesorting.go:102-115, ties by id)."""
    tot = {}
    for i in np.nonzero(member)[0]:
        m, c = tot.get(int(zone[i]), (0, 0))
        tot[int(zone[i])] = (m + int(meta[i][1]), c + int(meta[i][0]))
    zs = sorted(tot, key=lambda z: (tot[z][0], tot[z][1], z))
    return {z: p for p, z in enumerate(zs)}


def decide(meta, ff, over, zone, name_rank, member, cand, label_rank, exe, min_frag, hosting):
    """The arg-min of DESIGN.md §2.  meta / ff / over: lists of per-node (cpu, mem, gpu); member: kept by the scope; cand:
    member and schedulable and ready; hosting: set of node indices.  -> (winner index or -1, ambiguous)."""
    prio = zone_priority(meta, zone, member)
    rows = []
    for i in range(len(cand)):
        if not cand[i]:
            continue
        if min_frag:
            c = capacity(pyref.sub(meta[i], over[i]), exe)
            if c < 1:
                continue
            cls = 0 if i in hosting else 1
        else:
            if pyref.gt(exe, ff[i]):
                continue
            c, cls = 0, 0
        L = 0 if label_rank is None else (0x7fffffff if label_rank[i] < 0 else int(label_rank[i]))
        g = (cls, c, L, prio[int(zone[i])], int(meta[i][1]), int(meta[i][0]))
        rows.append((g, int(name_rank[i]), i))
    if not rows:
        return -1, False
    g, _, best = min(rows)
    amb = any(r[0] == g and int(meta[r[2]][2]) != int(meta[best][2]) for r in rows)
    return best, amb


def tie_permutations(order, key_of, gpu_of, name_of, limit=6):
    """Every executor order the reference's unstable sort may produce from `order` (SURVEY App. B6): within each run of
    nodes with equal (L, P, mem, cpu) -- which scheduleContextLessThan orders by name only when their gpu is equal too --
    every interleaving that keeps the name order of equal-gpu nodes.  One run permuted at a time (runs are contiguous and
    a decision only depends on the run holding its winner).  A run longer than `limit` is refused rather than skipped."""
    runs, s = [], 0
    for i in range(1, len(order) + 1):
        if i == len(order) or key_of(order[i]) != key_of(order[s]):
            if i - s > 1:
                runs.append((s, i))
            s = i
    for s, e in runs:
        if e - s > limit:
            raise ValueError("tie run of %d nodes: too long to enumerate" % (e - s))
        run = order[s:e]
        for perm in itertools.permutations(run):
            ok = all(not (gpu_of(a) == gpu_of(b) and name_of(a) > name_of(b))
                     for x, a in enumerate(perm) for b in perm[x + 1:])
            if ok and list(perm) != run:
                yield order[:s] + list(perm) + order[e:]
