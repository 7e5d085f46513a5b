"""The failover reconciler's node choice (EXT/failover.go:43-82, 286-436), three times: literally over oracle/pyref.py, literally in C
(tests/reconcile_oracle.c, string-keyed, exact), and as the closed form of DESIGN §2.3 with numpy (large cases).

A case is a dict:
  names[n], alloc (cpu, mem, gpu) int64 arrays, label[n] (instance-group label value, None = label missing), unschedulable[n],
  ready[n], creation[n] (int64, UnixNano), overhead (cpu, mem, gpu) or None, rows: res_node[r] (node index, -1 = a node not in
  the table), res (cpu, mem, gpu); drivers: dgroup[q] (label value the driver asks for, None = ""), exe (cpu, mem, gpu),
  min[q], running[q].
to_device_args() interns the label values into group ids and derives exe_count = max(0, Min - running) as a shim does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyref

HERE = os.path.dirname(os.path.abspath(__file__))
LIM = 1 << 61


# ---- literal restatement over pyref ---------------------------------------------------------------------------------------
def literal(case):
    """-> (placed[q], reserved node-name lists per driver, available dict name -> (cpu, mem, gpu) after the loop)."""
    names = case["names"]
    n = len(names)
    alloc = {names[i]: tuple(int(case["alloc"][d][i]) for d in range(3)) for i in range(n)}
    # :292-294 newest first; the node table is the lister order and Python's stable sort keeps it on ties, which is what Go
    # 1.19's pdqsort does for a lister that already returns the nodes newest first (DESIGN §2.3)
    nodes = sorted(range(n), key=lambda i: -int(case["creation"][i]))
    schedulable = {}                                                        # :296-314
    for i in nodes:
        if case["unschedulable"] is not None and case["unschedulable"][i]:
            continue
        if case["ready"] is not None and not case["ready"][i]:
            continue
        ig = case["label"][i] if case["label"][i] is not None else ""
        schedulable.setdefault(ig, []).append(names[i])
    usages = {}                                                             # :315 UsageForNodes (hard and soft rows alike)
    for r, node in enumerate(case["res_node"]):
        key = names[node] if node >= 0 else f"<not in the table {r}>"
        usages[key] = pyref.add(usages.get(key, pyref.ZERO), tuple(int(case["res"][d][r]) for d in range(3)))
    if case["overhead"] is not None:                                         # :316
        for i in range(n):
            usages[names[i]] = pyref.add(usages.get(names[i], pyref.ZERO), tuple(int(case["overhead"][d][i]) for d in range(3)))
    available = {g: {nm: pyref.sub(alloc[nm], usages.get(nm, pyref.ZERO)) for nm in ns} for g, ns in schedulable.items()}
    placed, reserved_names = [], []
    for i in range(len(case["min"])):
        g = case["dgroup"][i] if case["dgroup"][i] is not None else ""
        run = min(int(case["running"][i]), int(case["min"][i]))              # :141-143
        if g not in schedulable:                                            # :358-362
            placed.append(-1)
            reserved_names.append([])
            continue
        k = int(case["min"][i]) - run                                       # :366
        got, res = [], {}
        if k > 0:
            exe = tuple(int(case["exe"][d][i]) if case["exe"][d] is not None else 0 for d in range(3))
            got, res = find_nodes(k, exe, available[g], schedulable[g])
        for nm, r in res.items():                                           # :159
            available[g][nm] = pyref.sub(available[g][nm], r)
        placed.append(len(got))
        reserved_names.append(got)
    final = {nm: pyref.sub(alloc[nm], usages.get(nm, pyref.ZERO)) for nm in names}
    for g in available:
        final.update(available[g])
    return placed, reserved_names, final


def find_nodes(k, exe, available, ordered):
    """findNodes, EXT/failover.go:412-436."""
    out, reserved = [], {}
    for nm in ordered:
        if nm not in reserved:
            reserved[nm] = pyref.ZERO
        while True:
            reserved[nm] = pyref.add(reserved[nm], exe)
            if pyref.gt(reserved[nm], available[nm]):
                break
            out.append(nm)
            if len(out) == k:
                return out, reserved
    return out, reserved


# ---- what the device computes ----------------------------------------------------------------------------------------------
def to_device_args(case):
    """Interned groups in first-seen order over nodes then drivers, exe_count = max(0, Min - running)."""
    ids = {}
    for v in list(case["label"]) + list(case["dgroup"]):
        ids.setdefault(v if v is not None else "", len(ids))
    node_group = np.array([ids[v if v is not None else ""] for v in case["label"]], np.int32)
    dgroup = np.array([ids[v if v is not None else ""] for v in case["dgroup"]], np.int32)
    mn = np.asarray(case["min"], np.int64)
    count = (mn - np.minimum(np.asarray(case["running"], np.int64), mn)).clip(0).astype(np.int32)
    return node_group, dgroup, count, max(len(ids), 1)


def closed_form(case):
    """DESIGN §2.3 with numpy: -> (placed, executor_nodes CSR by the prefix sum of the counts, (cpu, mem, gpu) after, refused)."""
    node_group, dgroup, count, G = to_device_args(case)
    n = len(case["names"])
    av = np.stack([np.asarray(case["alloc"][d], np.int64) if case["alloc"][d] is not None else np.zeros(n, np.int64)
                   for d in range(3)]).astype(object)
    if case["overhead"] is not None:
        for d in range(3):
            if case["overhead"][d] is not None:
                av[d] -= np.asarray(case["overhead"][d], np.int64).astype(object)
    rn = np.asarray(case["res_node"], np.int64)
    for d in range(3):
        if case["res"][d] is None or len(rn) == 0:
            continue
        ok = rn >= 0
        np.add.at(av[d], rn[ok], -np.asarray(case["res"][d], np.int64)[ok].astype(object))
    av = av.astype(np.int64)          # exact while every input and sum stays in the int64 domain (tests keep it so)
    keep = np.ones(n, bool)
    if case["unschedulable"] is not None:
        keep &= ~np.asarray(case["unschedulable"], bool)
    if case["ready"] is not None:
        keep &= np.asarray(case["ready"], bool)
    creation = np.asarray(case["creation"], np.int64)
    order = np.lexsort((np.arange(n), ~creation, node_group))       # ~x = -x - 1: creation descending, without a wrap
    order = order[keep[order]]
    groups = {g: order[node_group[order] == g] for g in range(G)}
    exe = np.stack([np.asarray(case["exe"][d], np.int64) if case["exe"][d] is not None else np.zeros(len(count), np.int64)
                    for d in range(3)])
    off = np.zeros(len(count) + 1, np.int64)
    np.cumsum(count, out=off[1:])
    out = np.full(int(off[-1]), -1, np.int32)
    placed = np.zeros(len(count), np.int32)
    refused = False
    for i in range(len(count)):
        nodes = groups[int(dgroup[i])]
        k = int(count[i])
        if len(nodes) == 0:
            placed[i] = -1
            continue
        if k == 0:
            continue
        a = av[:, nodes]
        e = exe[:, i:i + 1]
        with np.errstate(divide="ignore"):
            cap = np.where(a < 0, 0, np.where(e == 0, k, a // np.where(e == 0, 1, e)))
        m = np.minimum(cap.min(axis=0), k)
        cs = np.cumsum(m)
        j = int(np.searchsorted(cs, k))          # first node whose inclusive sum reaches k
        if j < len(nodes):
            t = m[:j + 1].copy()
            t[j] = k - (cs[j - 1] if j else 0)
            charge = t + 1
            charge[j] = t[j]
            vis = nodes[:j + 1]
        else:
            t, charge, vis = m, m + 1, nodes
        placed[i] = int(t.sum())
        out[off[i]:off[i] + placed[i]] = np.repeat(vis, t)
        before = av[:, vis].astype(object)
        after = before - charge.astype(object)[None, :] * exe[:, i:i + 1].astype(object)
        refused |= bool(((before >= LIM) | (before <= -LIM) | (after <= -LIM)).any())
        av[:, vis] = np.clip(after, -(1 << 63), (1 << 63) - 1).astype(np.int64)
    return placed, out, off, (av[0], av[1], av[2]), refused


# ---- the C literal ---------------------------------------------------------------------------------------------------------
_clib = None


def c_lib():
    global _clib
    if _clib is None:
        d = tempfile.mkdtemp(prefix="reconcile_oracle_")
        so = os.path.join(d, "libreconcile_oracle.so")
        subprocess.check_call(["cc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "reconcile_oracle.c")])
        L = C.CDLL(so)
        L.orc_reconcile_find_nodes.restype = C.c_int
        L.orc_reconcile_find_nodes.argtypes = ([C.c_int32, C.c_void_p] + [C.c_void_p] * 3 + [C.c_void_p] * 4 + [C.c_void_p] * 3 +
                                               [C.c_int64, C.c_void_p] + [C.c_void_p] * 3 + [C.c_int32, C.c_void_p] + [C.c_void_p] * 3 +
                                               [C.c_void_p] * 2 + [C.c_void_p] * 5)
        _clib = L
    return _clib


def _strs(vals):
    arr = (C.c_char_p * max(len(vals), 1))()
    for i, v in enumerate(vals):
        arr[i] = None if v is None else v.encode()
    return arr


def c_literal(case):
    """-> (placed, executor node indices CSR by the prefix sum of max(0, Min - running), (cpu, mem, gpu) after, refused)."""
    return c_literal_bound(case)()


def c_literal_bound(case):
    """The C literal's arguments marshalled once -> a zero-argument callable that runs it (c_literal's result)."""
    L = c_lib()
    n, q = len(case["names"]), len(case["min"])
    i64 = lambda a: None if a is None else np.ascontiguousarray(a, np.int64)
    p = lambda a: None if a is None else a.ctypes.data
    alloc = [i64(a) for a in case["alloc"]]
    over = [i64(a) for a in case["overhead"]] if case["overhead"] is not None else [None] * 3
    res = [i64(a) for a in case["res"]]
    exe = [i64(a) for a in case["exe"]]
    names = _strs(case["names"])
    labels = _strs(case["label"])
    rn = [case["names"][v] if v >= 0 else f"<not in the table {r}>" for r, v in enumerate(case["res_node"])]
    rnames = _strs(rn)
    dg = _strs(case["dgroup"])
    fu = None if case["unschedulable"] is None else np.ascontiguousarray(case["unschedulable"], np.uint8)
    fr = None if case["ready"] is None else np.ascontiguousarray(case["ready"], np.uint8)
    cr = i64(case["creation"])
    mn = np.ascontiguousarray(case["min"], np.int32)
    run = np.ascontiguousarray(case["running"], np.int32)
    _, _, count, _ = to_device_args(case)
    off = np.zeros(q + 1, np.int64)
    np.cumsum(count, out=off[1:])
    placed = np.zeros(max(q, 1), np.int32)
    out = np.full(max(int(off[-1]), 1), -1, np.int32)
    av = [np.zeros(max(n, 1), np.int64) for _ in range(3)]

    def call(_keep=(alloc, over, res, exe, names, labels, rnames, dg, fu, fr, cr, mn, run)):
        bad = L.orc_reconcile_find_nodes(n, names, p(alloc[0]), p(alloc[1]), p(alloc[2]), labels, p(fu), p(fr), p(cr),
                                         p(over[0]), p(over[1]), p(over[2]), len(rn), rnames, p(res[0]), p(res[1]), p(res[2]),
                                         q, dg, p(exe[0]), p(exe[1]), p(exe[2]), p(mn), p(run),
                                         p(placed), p(out), p(av[0]), p(av[1]), p(av[2]))
        return placed[:q].copy(), out[:int(off[-1])].copy(), off, tuple(a[:n].copy() for a in av), bool(bad)
    return call


# ---- random cases ----------------------------------------------------------------------------------------------------------
def random_case(rng, n_nodes, n_groups, n_drivers, n_rows, big=False):
    """Creation ties, unschedulable / not-ready nodes, the "" group (label missing), groups without nodes, negative
    availabilities, zero-dimension and all-zero executors, k = 0, exact-capacity completions and partial placements."""
    labels = [None] + [f"ig-{g}" for g in range(1, n_groups)]
    gsel = rng.integers(0, n_groups, n_nodes)
    label = [labels[g] for g in gsel]
    cpu = rng.integers(0, 64, n_nodes) * 1000
    mem = rng.integers(0, 256, n_nodes) << 30
    gpu = np.where(rng.random(n_nodes) < 0.3, rng.integers(0, 8, n_nodes), 0)
    creation = rng.integers(0, max(2, n_nodes // 3), n_nodes).astype(np.int64) * 1_000_000_000   # many ties
    unsched = (rng.random(n_nodes) < 0.1).astype(np.uint8)
    ready = (rng.random(n_nodes) > 0.1).astype(np.uint8)
    over = (rng.integers(0, 2000, n_nodes), rng.integers(0, 4, n_nodes) << 30, np.zeros(n_nodes, np.int64))
    res_node = rng.integers(-1, n_nodes, n_rows).astype(np.int32)                 # -1: a reservation on a node not in the table
    res = (rng.integers(0, 16, n_rows) * 1000, rng.integers(0, 64, n_rows) << 30, rng.integers(0, 2, n_rows))
    dlabels = labels + ["ig-missing"]
    dgroup = [dlabels[g] for g in rng.integers(0, len(dlabels), n_drivers)]      # interleaved groups, some without nodes
    shape = rng.integers(0, 6, n_drivers)
    ecpu = np.where(shape == 0, 0, rng.integers(1, 8, n_drivers) * 500)
    emem = np.where(shape == 1, 0, rng.integers(1, 32, n_drivers) << 30)
    egpu = np.where(shape == 2, rng.integers(1, 3, n_drivers), 0)
    allzero = shape == 3
    ecpu, emem, egpu = np.where(allzero, 0, ecpu), np.where(allzero, 0, emem), np.where(allzero, 0, egpu)
    if big:
        huge = rng.random(n_drivers) < 0.3
        ecpu = np.where(huge, (1 << 59) + rng.integers(0, 1 << 20, n_drivers), ecpu)
    mn = rng.integers(0, 40, n_drivers)
    running = np.where(rng.random(n_drivers) < 0.3, rng.integers(0, 50, n_drivers), 0)
    return dict(names=[f"node-{i:06d}" for i in range(n_nodes)], alloc=(cpu, mem, gpu), label=label, unschedulable=unsched,
                ready=ready, creation=creation, overhead=over, res_node=res_node, res=res, dgroup=dgroup, exe=(ecpu, emem, egpu),
                min=mn, running=running)


def literal_flat(case):
    """literal() as arrays: (placed, executor node indices CSR by the prefix sum of the counts, (cpu, mem, gpu) after)."""
    placed, got, final = literal(case)
    index = {nm: i for i, nm in enumerate(case["names"])}
    _, _, count, _ = to_device_args(case)
    off = np.zeros(len(count) + 1, np.int64)
    np.cumsum(count, out=off[1:])
    out = np.full(int(off[-1]), -1, np.int32)
    for i, g in enumerate(got):
        out[off[i]:off[i] + len(g)] = [index[nm] for nm in g]
    av = tuple(np.array([final[nm][d] for nm in case["names"]], dtype=object) for d in range(3))
    return np.array(placed, np.int32), out, off, av
