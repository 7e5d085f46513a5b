"""The unschedulable-pod marker's capacity check, twice: literally, and as the criterion of DESIGN §2.2.

literal_exceeds() is DoesPodExceedClusterCapacity (EXT/unschedulablepods.go:132-166) over oracle/pyref.py: zero-usage metadata
from NodeSchedulingMetadataForNodes, the affinity nodes in the given (lister) order as both priority orders, one packer.
model_exceeds() is what gp_exceeds_cluster_capacity computes: T = sum min(cap(n|0), C), M = max over the nodes the driver fits
on of min(cap(d|drv), C) - min(cap(d|0), C), per zone for the single-AZ packers, plus the positivity rule of chooseBestResult.
"""
from __future__ import annotations

from oracle import pyref

C = 1 << 31
PACKERS = ("tightly-pack", "distribute-evenly", "az-aware-tightly-pack", "single-az-tightly-pack", "single-az-minimal-fragmentation")


def _cap(avail, reserved, exe):
    return min(pyref._capacity_single_dimension(avail[d], reserved[d], exe[d]) for d in range(3))


def literal_exceeds(packer, alloc, overhead, zones, names, drv, exe, k):
    """alloc / overhead: name -> (cpu, mem, gpu) over ALL nodes; names: the driver's affinity nodes in lister order;
    zones: name -> ZoneLabel.  -> True when the driver exceeds cluster capacity."""
    sub_alloc = {n: alloc[n] for n in names}
    meta, sched = pyref.node_scheduling_metadata(sub_alloc, overhead, [])
    order = list(names)
    if packer in ("tightly-pack", "distribute-evenly"):
        dist = pyref.tightly_pack_executors if packer == "tightly-pack" else pyref.distribute_executors_evenly
        ok = pyref.spark_bin_pack(drv, exe, k, order, order, meta, dist)[2]
    elif packer == "az-aware-tightly-pack":
        ok = pyref.az_aware_tightly_pack(drv, exe, k, order, order, meta, sched, zones)[2]
    elif packer == "single-az-tightly-pack":
        ok = pyref.single_az_tightly_pack(drv, exe, k, order, order, meta, sched, zones)[2]
    elif packer == "single-az-minimal-fragmentation":
        ok = pyref.single_az_minimal_fragmentation(drv, exe, k, order, order, meta, sched, zones)[2]
    else:
        raise ValueError(packer)
    return not ok


def zone_terms(sched_list, drv, exe):
    """[(zone, schedulable)] -> {zone: (T_z, M_z)} with M_z = None when the driver fits on no node of the zone."""
    out = {}
    for z, s in sched_list:
        c0 = min(_cap(s, pyref.ZERO, exe), C)
        t, m = out.get(z, (0, None))
        t += c0
        if not pyref.gt(drv, s):
            delta = min(_cap(s, drv, exe), C) - c0
            m = delta if m is None else max(m, delta)
        out[z] = (t, m)
    return out


def positive_efficiency(packer, drv, exe, k):
    """chooseBestResult keeps a zone only when AvgPackingEfficiency.Max > 0: some entry of [driver] + ExecutorNodes reserves a
    positive amount (minimal fragmentation never adds its executors to `reserved`)."""
    drv_nz = any(v != 0 for v in drv)
    if packer == "single-az-minimal-fragmentation":
        return drv_nz
    return drv_nz or (k >= 1 and any(v != 0 for v in exe))


def model_exceeds(packer, sched_list, drv, exe, k):
    """sched_list: [(zone, schedulable)] of the driver's affinity nodes (any order)."""
    terms = zone_terms(sched_list, drv, exe)
    if packer in ("tightly-pack", "distribute-evenly", "az-aware-tightly-pack"):
        ms = [m for _, m in terms.values() if m is not None]
        if not ms:
            return True
        return sum(t for t, _ in terms.values()) + max(ms) < k
    if not positive_efficiency(packer, drv, exe, k):
        return True
    return not any(m is not None and t + m >= k for t, m in terms.values())


def boundary_k(sched_list, drv, exe):
    """T + M over the whole set (None when no driver fits): the count at which tightly-pack flips."""
    terms = zone_terms(sched_list, drv, exe)
    ms = [m for _, m in terms.values() if m is not None]
    return None if not ms else sum(t for t, _ in terms.values()) + max(ms)


# ---- vectorised form for large clusters (same criterion) ------------------------------------------------------------------
NONE = -(1 << 63)


def np_caps(cols, exe):
    """min(cap(n|0), C) per node; cols = [cpu, mem, gpu] int64 arrays of the schedulable (or remaining) resources."""
    import numpy as np
    out = np.full(len(cols[0]), C, np.int64)
    for d in range(3):
        a = cols[d]
        q = np.full(len(a), C, np.int64) if exe[d] == 0 else np.minimum(np.maximum(a, 0) // exe[d], C)
        out = np.minimum(out, np.where(a < 0, 0, q))
    return out


def np_zone_terms(cols, zone, n_zones, drv, exe):
    """-> (T[z], M[z]) int64 arrays, M = NONE where the driver fits on no node of zone z."""
    import numpy as np
    c0 = np_caps(cols, exe)
    fits = (cols[0] >= drv[0]) & (cols[1] >= drv[1]) & (cols[2] >= drv[2])
    cd = np_caps([cols[d] - drv[d] for d in range(3)], exe)
    delta = np.where(fits, cd - c0, NONE)
    T = np.zeros(n_zones, np.int64)
    np.add.at(T, zone, c0)
    M = np.full(n_zones, NONE, np.int64)
    np.maximum.at(M, zone, delta)
    return T, M


def np_decide(packer, T, M, drv, exe, k):
    """exceeds for count k from the per-zone terms of the driver's node set."""
    has_fit = M > NONE
    if packer in ("tightly-pack", "distribute-evenly", "az-aware-tightly-pack"):
        return not has_fit.any() or int(T.sum()) + int(M[has_fit].max()) < k
    if not positive_efficiency(packer, drv, exe, k):
        return True
    return not has_fit.any() or int((T[has_fit] + M[has_fit]).max()) < k
