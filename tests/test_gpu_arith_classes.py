"""Every capacity-arithmetic class of every kernel family at the class boundaries, on the device.

Part A: small snapshots whose per-dimension maximum sits at 2^(32+t) - 1, 2^(32+t) and 2^(32+t) + 1 (where the fast class
and the compact view's shift switch), nodes at multiples of the requests and one off, requests of every divider kind,
drivers equal to a node's availability, counts around the exact capacity, the uint16 capacity cache and the table clamp;
run through every entry point and compared with the closed-form oracle, the literal C and the Python references.  The model
of tests/arith_class_model.py says which class and divider kinds each application takes; the coverage matrix it builds
must hit every reachable cell.
Part B: scaling cpu, memory and gpu by their own factors leaves every capacity and every driver-fit test unchanged, so
every decision must be bit-identical to the unscaled run's, at full size and across classes.
Part C: usage deltas that raise the memory maximum across a shift boundary of a long-lived context, then packs of every
kind on it, each against a fresh context built from its snapshot and against the oracle."""
import os

import numpy as np
import pytest

import arith_class_model as m
import capacity_ref as cr
import reconcile_ref as R
import reschedule_ref as rr
from helpers import assert_same_results, group_slices, literal_batch, node_names, res_aos
from oracle import pyref
from test_gpu_az_aware_batch import ORC_AZ_AWARE, az_layout

pytestmark = pytest.mark.gpu
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
MF_DEV, MF_ORC = 2, 4
GI = 1 << 30


def make_packer(gangpack, **env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return gangpack.GangPacker()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def ctxs(gangpack):
    ps = {"default": make_packer(gangpack), "tables0": make_packer(gangpack, GANGPACK_TABLES=0),
          "warp0": make_packer(gangpack, GANGPACK_FIFO_WARP=0)}
    yield ps
    for p in ps.values():
        p.close()


# ---------------------------------------------------------------------------------------------------------------------
# coverage: family x class x divider kind x gpu state, from the model
# ---------------------------------------------------------------------------------------------------------------------
IDLE, USED = "gpu idle", "gpu used"
ALL = set(m.KINDS)
FASTK = {m.INF, m.MAGIC2, m.MAGIC}


DIMDIV = ("resched", "resched_res", "reconcile")      # the make_dimdiv users
FAMILIES = ("scan", "minfrag", "fifo", "marker") + DIMDIV


def _cells(family, cls_kinds):
    return {(family, c, k, g) for (c, g), ks in cls_kinds.items() for k in ks}


REACHABLE = (
    _cells("scan", {(m.FAST32, IDLE): FASTK, (m.FAST64, IDLE): FASTK, (m.GENERAL, IDLE): ALL, (m.GENERAL, USED): ALL})
    | _cells("minfrag", {(m.FAST32, IDLE): FASTK, (m.GENERAL, IDLE): ALL, (m.GENERAL, USED): ALL})
    | _cells("fifo", {(m.FAST64, IDLE): FASTK, (m.FAST64, USED): FASTK | {m.SHIFT}, (m.GENERAL, IDLE): ALL, (m.GENERAL, USED): ALL})
    | _cells("marker", {(m.GENERAL, IDLE): ALL, (m.GENERAL, USED): ALL})
    | {c for fam in DIMDIV for c in _cells(fam, {(m.GENERAL, IDLE): ALL - {m.MAGIC2}, (m.GENERAL, USED): ALL - {m.MAGIC2}})})


def note(cov, family, apps, meta):
    """Count the (family, class, divider kind, gpu state) cells of the applications `apps` just checked through `family`."""
    q = len(apps["count"])
    for i in range(q):
        app = m.App((int(apps["drv_cpu"][i]), int(apps["drv_mem"][i]), int(apps["drv_gpu"][i])),
                    (int(apps["exe_cpu"][i]), int(apps["exe_mem"][i]), int(apps["exe_gpu"][i])), int(apps["count"][i]))
        g = USED if m.uses_gpu(app, meta) else IDLE
        if family in DIMDIV:
            cls, kinds = m.GENERAL, [m.kind_name(m.make_dimdiv(e)) for e in app.exe]
        elif family == "marker":
            cls, kinds = m.GENERAL, [m.kind_name(m.prep_dim(e, t, 0)[0]) for t, e in enumerate(app.exe)]
        else:
            cls = m.family_class(family, app, meta)
            kinds = [m.kind_name(m.prep_dim(e, t, meta.max_avail[t])[0]) for t, e in enumerate(app.exe)]
        for k in set(kinds):
            cov[(family, cls, k, g)] = cov.get((family, cls, k, g), 0) + 1


# ---------------------------------------------------------------------------------------------------------------------
# Part A: the boundary lattice
# ---------------------------------------------------------------------------------------------------------------------
def boundary_values(mx, es):
    """Availabilities q*e - 1, q*e, q*e + 1 for the requests `es`, kept in [0, mx], plus mx itself."""
    out = {mx, max(mx - 1, 0), mx // 2}
    for e in es:
        for q in (1, 2, 3, (1 << 16) - 1):
            for d in (-1, 0, 1):
                v = q * e + d
                if 0 <= v <= mx:
                    out.add(v)
    return sorted(out)


def lattice_requests(s, cpu_small):
    """Executor memory / cpu requests of every divider kind around the view shift s of memory."""
    mem = {0, 1, 2, 3, 1 << 20, 3 << 20, (1 << 32) - 1, (1 << 32) + 1, ((1 << 33) - 1) << 3, 12345678901}
    for j in (s - 1, s, s + 1, s + 2, s + 31, s + 32, s + 33):
        if j >= 0:
            mem.update(x for x in ((1 << j), 3 << j, ((1 << 32) - 1) << j) if 0 < x < m.MAX_QUANTITY)
    cpu = [1000, 3, 1, 0, 250, (1 << 32) - 1]
    if cpu_small:
        # shift >= S0 + 32 with S0 = 0: the fast class without the compact view (pack_app_fast64).  Such a request exceeds every
        # availability of the snapshot (max >> sh < 2^32 forces sh >= S0), so these applications reach the scan's fast64
        # path with capacity 0 only; the FIFO kernels divide every fast request with fast_q_magic, nonzero quotients included.
        cpu += [1 << 33, 3 << 32]
    return sorted(mem), cpu


def lattice_case(rng, t, d, gpu_state, cpu_t=None, cpu_e=None):
    """-> (cpu, mem, gpu, apps, meta): about 40 nodes whose memory maximum is 2^(32+t) + d."""
    mx = (1 << (32 + t)) + d
    s = m.shift_for(mx)
    mem_e, lat_cpu = lattice_requests(s, cpu_t is None)
    cpu_e = lat_cpu if cpu_e is None else cpu_e
    mem_nodes = boundary_values(mx, [3 << 20, 1 << max(s, 1), 3 << s, (1 << 32) - 1, 1 << 30])
    mem_nodes = list(rng.choice(mem_nodes, min(len(mem_nodes), 36), replace=False)) + [mx]
    n = len(mem_nodes)
    cmx = 96000 if cpu_t is None else (1 << (32 + cpu_t[0])) + cpu_t[1]
    cpu = np.array(boundary_values(cmx, [1000, 3, 250])[-n:], np.int64)
    if len(cpu) < n:
        cpu = np.resize(cpu, n)
    cpu = rng.permutation(cpu)
    cpu[0] = cmx
    mem = np.array(mem_nodes, np.int64)
    gpu = np.zeros(n, np.int64)
    if gpu_state == "used":
        gpu = rng.integers(0, 5, n).astype(np.int64)
    elif gpu_state == "negative":
        gpu[int(rng.integers(0, n))] = -1
    cpu[1] = -1                                           # a negative cpu availability
    meta = m.SnapMeta(cpu, mem, gpu)
    rows = []
    for em in mem_e:
        for ec in cpu_e:
            rows.append((ec, em))
    rng.shuffle(rows)
    q = len(rows)
    a = {k: np.zeros(q, np.int64) for k in KEYS}
    a["count"] = np.zeros(q, np.int32)
    big = 0
    for i, (ec, em) in enumerate(rows):
        eg = int(rng.choice([0, 1, 2, 3])) if gpu_state == "used" else 0
        v = i % 4
        if v == 1:                                        # a driver equal to a node's availability
            j = int(rng.integers(0, n))
            drv = (max(int(cpu[j]), 0), int(mem[j]), max(int(gpu[j]), 0))
        elif v == 2:
            drv = (1000, 1 << 30, 1 if gpu_state == "used" else 0)
        else:
            drv = (0, 0, 0)
        exe = (ec, em, eg)
        caps = [m.node_cap((int(cpu[x]), int(mem[x]), int(gpu[x])), (0, 0, 0), exe) for x in range(n)]
        total = None if any(c is None for c in caps) else sum(caps)
        if total is not None and total <= 3000:
            k = max(0, total + (i % 3) - 1)                  # cap - 1, cap, cap + 1
        elif big < 4 and total is not None and total >= (1 << 16) + 2:
            k = ((1 << 16) - 1, 1 << 16)[big % 2]            # the uint16 capacity cache's boundary
            big += 1
        else:
            k = int(rng.integers(0, 40))
        for key, val in zip(("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu"), drv + exe):
            a[key][i] = val
        a["count"][i] = k
    return cpu, mem, gpu, a, meta


def _closed(oracle, algo, mode, cpu, mem, gpu, dorder, eorder, a, young=None):
    drv = res_aos(a["drv_cpu"], a["drv_mem"], a["drv_gpu"]); exe = res_aos(a["exe_cpu"], a["exe_mem"], a["exe_gpu"])
    _, dn, en, off, final = oracle.closed_batch(algo, mode, cpu, mem, gpu, dorder, eorder, drv, exe, a["count"], young,
                                                n_threads=8 if mode == 0 else 1)
    return (dn, en, off), final


def pyref_batch(algo, cpu, mem, gpu, dorder, eorder, a):
    """oracle/pyref.py in Python integers: (driver_node, executor_nodes, off)."""
    names = node_names(len(cpu))
    meta = {names[i]: (int(cpu[i]), int(mem[i]), int(gpu[i])) for i in range(len(cpu))}
    dist = (pyref.tightly_pack_executors, pyref.distribute_executors_evenly, pyref.minimal_fragmentation)[algo]
    q = len(a["count"])
    off = np.zeros(q + 1, np.int64); np.cumsum(a["count"], out=off[1:])
    dn = np.full(q, -1, np.int32); en = np.full(max(int(off[-1]), 1), -1, np.int32)
    idx = {nm: i for i, nm in enumerate(names)}
    for i in range(q):
        drv = tuple(int(a[k][i]) for k in ("drv_cpu", "drv_mem", "drv_gpu"))
        exe = tuple(int(a[k][i]) for k in ("exe_cpu", "exe_mem", "exe_gpu"))
        d, nodes, ok = pyref.spark_bin_pack(drv, exe, int(a["count"][i]), [names[j] for j in dorder], [names[j] for j in eorder],
                                            meta, dist)
        if ok:
            dn[i] = idx[d]
            en[off[i]:off[i + 1]] = [idx[x] for x in nodes]
    return dn, en, off


LATTICE = [(t, d, g) for t in (0, 4, 12) for d in (-1, 0, 1) for g in ("idle", "used", "negative")]
CPU_SWITCH = [(0, -1), (0, 0), (0, 1)]
CPU_SWITCH_REQUESTS = [1000, 3, (1 << 31) + 1, 2, 1 << 20, 3 << 10, (1 << 32) - 1, 1]
CASES = {}          # case -> coverage of that case's entry calls, recorded once the case has passed


def _fifo_zone_check(oracle, p, oalgo, fn, args, cpu, mem, gpu, sched, names, zone_of, dorder, eorder, fa, mode, label):
    """One zone FIFO entry against the literal C (efficiencies on): every decision and the final snapshot."""
    cl = oracle.Cluster(names, cpu, mem, gpu, sched=sched, zone=["zone-%d" % z for z in zone_of])
    drv = res_aos(fa["drv_cpu"], fa["drv_mem"], fa["drv_gpu"]); exe = res_aos(fa["exe_cpu"], fa["exe_mem"], fa["exe_gpu"])
    _, wd, we, woff = cl.fifo(oalgo, mode, drv, exe, fa["count"], fa["young"], [names[i] for i in dorder],
                              [names[i] for i in eorder], with_efficiencies=True)
    zone, gd, ge, goff, _ = fn(fa, *args)
    assert_same_results((gd, ge, goff), (wd, we, woff), label)
    for x, y in zip(p.get_snapshot(), cl.available()):
        assert np.array_equal(x, y), label + " final snapshot"


def run_lattice_case(oracle, ctxs, cpu, mem, gpu, a, meta, rng, label, small=False, full=True):
    """Every entry point on one boundary snapshot against its references -> the coverage of the calls that were checked."""
    cov = {}
    n = len(cpu)
    eorder = rng.permutation(n).astype(np.int32)
    dorder = np.concatenate([rng.permutation(n)[: n // 2], eorder[:3]]).astype(np.int32)
    dorder = np.unique(dorder)[rng.permutation(len(np.unique(dorder)))].astype(np.int32)
    # ---- independent: tightly-pack, distribute-evenly, minimal-fragmentation on every context
    for algo in (0, 1, 2):
        want, _ = _closed(oracle, MF_ORC if algo == 2 else algo, 0, cpu, mem, gpu, dorder, eorder, a)
        lit = literal_batch(oracle, MF_ORC if algo == 2 else algo, cpu, mem, gpu, dorder, eorder, a)
        assert_same_results(lit, want, f"{label} literal vs closed algo {algo}")
        if small:
            sel = np.nonzero(a["count"] <= 3000)[0]
            sub = {k: v[sel] for k, v in a.items()}
            assert_same_results(pyref_batch(algo, cpu, mem, gpu, dorder, eorder, sub),
                                _closed(oracle, MF_ORC if algo == 2 else algo, 0, cpu, mem, gpu, dorder, eorder, sub)[0],
                                f"{label} pyref algo {algo}")
        for name in ("default", "tables0", "warp0"):
            p = ctxs[name]
            p.set_snapshot(cpu, mem, gpu, eorder, dorder)
            got = p.pack_batch(a, algo, 0)
            assert_same_results(got, want, f"{label} {name} algo {algo}")
            if algo < 2:
                w = p.pack_batch(a, algo, 0, wire=dict(quantity_bits=64, node_bits=16, offsets=False))
                assert_same_results((w[0], w[1].astype(np.int32), w[2]), want, f"{label} {name} wire algo {algo}")
        for i in range(0, len(a["count"]), 23):         # the single-application entry
            ok, dn, ex = ctxs["default"].pack_one(algo, (a["drv_cpu"][i], a["drv_mem"][i], a["drv_gpu"][i]),
                                                  (a["exe_cpu"][i], a["exe_mem"][i], a["exe_gpu"][i]), int(a["count"][i]))
            assert ok == (want[0][i] >= 0), (label, algo, i)
            if ok:
                assert dn == want[0][i] and np.array_equal(ex, want[1][want[2][i]:want[2][i + 1]]), (label, algo, i)
        note(cov, "minfrag" if algo == 2 else "scan", a, meta)
    # ---- FIFO: reference and exact accounting, warp-first and CTA-only contexts, the final snapshot
    young = (rng.random(len(a["count"])) < 0.7).astype(np.uint8)
    fa = dict(a, young=young)
    for mode in (1, 2):
        for algo in (0, 1):
            want, final = _closed(oracle, algo, mode, cpu, mem, gpu, dorder, eorder, a, young)
            for name in ("default", "warp0"):
                p = ctxs[name]
                p.set_snapshot(cpu, mem, gpu, eorder, dorder)
                got = p.pack_batch(fa, algo, mode)
                assert_same_results(got, want, f"{label} {name} fifo algo {algo} mode {mode}")
                for x, y in zip(p.get_snapshot(), final):
                    assert np.array_equal(x, y), (label, name, algo, mode)
    note(cov, "fifo", a, meta)
    if not full:
        return cov
    # ---- zone packers: two zones, against the literal C with efficiencies
    zone_of = np.arange(n) % 2
    names = node_names(n)
    sched = (np.maximum(cpu, 0) + 1000, mem + (1 << 20), np.maximum(gpu, 0) + 1)
    labels = ["zone-%d" % z for z in zone_of]
    drv = res_aos(a["drv_cpu"], a["drv_mem"], a["drv_gpu"]); exe = res_aos(a["exe_cpu"], a["exe_mem"], a["exe_gpu"])
    p = ctxs["default"]
    zones, eo, do, eoff, doff = az_layout(dorder, eorder, zone_of)
    Zn = len(zones)
    single = (eo[:eoff[Zn]], do[:doff[Zn]], eoff[:Zn + 1], doff[:Zn + 1])
    for algo, oalgo in ((0, 2), (2, 5)):                 # single-az-tightly-pack / -minimal-fragmentation
        cl = oracle.Cluster(names, cpu, mem, gpu, sched=sched, zone=labels)
        wd, we, woff = cl.binpack_batch(oalgo, drv, exe, a["count"], [names[i] for i in dorder], [names[i] for i in eorder],
                                        with_efficiencies=True, n_threads=4)
        p.set_snapshot(cpu, mem, gpu, *single)
        p.set_schedulable(*sched)
        assert_same_results(p.pack_batch_zones(a, algo)[1:4], (wd, we, woff), f"{label} zones algo {algo}")
        for mode in (1, 2):
            p.set_snapshot(cpu, mem, gpu, *single)
            p.set_schedulable(*sched)
            _fifo_zone_check(oracle, p, oalgo, p.pack_fifo_zones, (algo, mode), cpu, mem, gpu, sched, names, zone_of, dorder,
                             eorder, fa, mode, f"{label} fifo zones algo {algo} mode {mode}")
    cl = oracle.Cluster(names, cpu, mem, gpu, sched=sched, zone=labels)
    wd, we, woff = cl.binpack_batch(ORC_AZ_AWARE, drv, exe, a["count"], [names[i] for i in dorder], [names[i] for i in eorder],
                                    with_efficiencies=True, n_threads=4)
    p.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
    p.set_schedulable(*sched)
    assert_same_results(p.pack_batch_az_aware(a, eorder, dorder, len(zones))[1:4], (wd, we, woff), f"{label} az-aware")
    for mode in (1, 2):
        p.set_snapshot(cpu, mem, gpu, eo, do, eoff, doff)
        p.set_schedulable(*sched)
        _fifo_zone_check(oracle, p, ORC_AZ_AWARE, p.pack_fifo_az_aware, (mode, eorder, dorder, len(zones)), cpu, mem, gpu, sched,
                         names, zone_of, dorder, eorder, fa, mode, f"{label} fifo az-aware mode {mode}")
    # ---- the marker: exceeds-cluster-capacity at the flip count, against the criterion in Python integers
    sn = [(0, (int(cpu[x]), int(mem[x]), int(gpu[x]))) for x in range(n)]
    ka = {k: a[k].copy() for k in KEYS}
    for i in range(len(ka["count"])):
        drv_i = (int(a["drv_cpu"][i]), int(a["drv_mem"][i]), int(a["drv_gpu"][i]))
        exe_i = (int(a["exe_cpu"][i]), int(a["exe_mem"][i]), int(a["exe_gpu"][i]))
        b = cr.boundary_k(sn, drv_i, exe_i)
        if b is not None and 0 <= b + 1 < (1 << 31) - 1:
            ka["count"][i] = max(0, b + (i % 3) - 1)
    ka["count"] = np.minimum(ka["count"], (1 << 31) - 1).astype(np.int32)
    ka["group"] = np.zeros(len(ka["count"]), np.int32)
    alloc = (np.maximum(cpu, 0), mem, np.maximum(gpu, 0))
    over = (alloc[0] - cpu, np.zeros(n, np.int64), alloc[2] - gpu)          # schedulable = the snapshot, negatives included
    for bp in (0, 3):
        got = p.exceeds_cluster_capacity(alloc, ka, bp, overhead=over)
        for i in range(len(ka["count"])):
            drv_i = (int(ka["drv_cpu"][i]), int(ka["drv_mem"][i]), int(ka["drv_gpu"][i]))
            exe_i = (int(ka["exe_cpu"][i]), int(ka["exe_mem"][i]), int(ka["exe_gpu"][i]))
            assert bool(got[i]) == cr.model_exceeds(cr.PACKERS[bp], sn, drv_i, exe_i, int(ka["count"][i])), (label, bp, i)
    note(cov, "marker", ka, meta)
    # ---- make_dimdiv users: reschedule (first fit / minimal fragmentation), the same from reservations, the reconciler
    p.set_snapshot(cpu, mem, gpu, eorder, eorder)
    ec, em, eg = a["exe_cpu"], a["exe_mem"], a["exe_gpu"]
    ff = p.reschedule_executors((ec, em, eg))
    mf = p.reschedule_executors((ec, em, eg), min_frag=True)
    onames = [names[i] for i in eorder]
    rcl = oracle.Cluster(names, cpu, mem, gpu)
    for i in range(len(ec)):
        e_i = (int(ec[i]), int(em[i]), int(eg[i]))
        w = rcl.reschedule_executor(False, e_i, onames)
        assert ff[i] == (names.index(w) if w else -1), (label, "first fit", i)
        w = rcl.reschedule_executor(True, e_i, onames)
        assert mf[i] == (names.index(w) if w else -1), (label, "min frag", i)
    note(cov, "resched", a, meta)
    # from the reservations: allocatable = the snapshot clipped at 0, one reservation row per negative node restores it
    neg = np.nonzero((cpu < 0) | (gpu < 0))[0]
    rnode = neg.astype(np.int32)
    rres = (alloc[0][neg] - cpu[neg], np.zeros(len(neg), np.int64), alloc[2][neg] - gpu[neg])
    host = [[int(x) for x in rng.integers(0, n, int(rng.integers(0, 4)))] for _ in range(len(ec))]
    zid, rank = np.zeros(n, np.int32), np.arange(n, dtype=np.int32)
    tri = [(int(cpu[x]), int(mem[x]), int(gpu[x])) for x in range(n)]
    for min_frag in (False, True):
        got, amb = p.reschedule_from_reservations(alloc, None, rnode, rres, (ec, em, eg), min_frag=min_frag,
                                                  hosting=host if min_frag else None, zone_id=zid, n_zones=1, name_rank=rank)
        for i in range(len(ec)):
            e_i = (int(ec[i]), int(em[i]), int(eg[i]))
            w, am = rr.decide(tri, tri, [(0, 0, 0)] * n, zid, rank, [True] * n, [True] * n, None, e_i, min_frag,
                              set(host[i]) if min_frag else set())
            assert (got[i], bool(amb[i])) == (w, am), (label, "from reservations", min_frag, i)
    note(cov, "resched_res", a, meta)
    case = dict(names=names, alloc=alloc, label=["ig"] * n, unschedulable=None,
                ready=None, creation=rng.integers(0, 5, n).astype(np.int64), overhead=None, res_node=rnode,
                res=rres, dgroup=["ig"] * len(ec), exe=(ec, em, eg),
                min=np.minimum(a["count"], 5000).astype(np.int64), running=np.zeros(len(ec), np.int64))
    ng, dg, count, G = R.to_device_args(case)
    got = p.reconcile_find_nodes(case["alloc"], None, case["res_node"], case["res"], ng, case["creation"],
                                 dict(exe_cpu=ec, exe_mem=em, exe_gpu=eg, count=count, group=dg), G)
    want = R.closed_form(case)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2]), label
    for i in np.nonzero(want[0] > 0)[0]:
        assert np.array_equal(got[1][want[2][i]:want[2][i] + want[0][i]], want[1][want[2][i]:want[2][i] + want[0][i]]), (label, i)
    for dd in range(3):
        assert np.array_equal(got[3][dd], want[3][dd]), (label, dd)
    note(cov, "reconcile", a, meta)
    return cov


def run_case(oracle, ctxs, key):
    if key[0] == "lattice":
        _, t, d, gpu_state = key
        rng = np.random.default_rng(1000 * t + 10 * (d + 1) + ("idle", "used", "negative").index(gpu_state))
        cpu, mem, gpu, a, meta = lattice_case(rng, t, d, gpu_state)
        return run_lattice_case(oracle, ctxs, cpu, mem, gpu, a, meta, rng, f"t={t} d={d} gpu {gpu_state}", small=(t, d) == (0, 0))
    cpu_t = key[1]
    rng = np.random.default_rng(77 + cpu_t[1])
    cpu, mem, gpu, a, meta = lattice_case(rng, 0, -1, "idle", cpu_t=cpu_t, cpu_e=CPU_SWITCH_REQUESTS)
    return run_lattice_case(oracle, ctxs, cpu, mem, gpu, a, meta, rng, f"cpu maximum {cpu_t}", full=False)


@pytest.mark.parametrize("t,d,gpu_state", LATTICE)
def test_boundary_lattice(oracle, ctxs, t, d, gpu_state):
    CASES[("lattice", t, d, gpu_state)] = run_case(oracle, ctxs, ("lattice", t, d, gpu_state))


@pytest.mark.parametrize("cpu_t", CPU_SWITCH)
def test_cpu_maximum_at_the_switch(oracle, ctxs, cpu_t):
    """The cpu dimension's maximum at 2^32 - 1, 2^32, 2^32 + 1 (memory far below its own switch), requests of every kind in
    cpu; independent packing on the table and scan contexts and FIFO with the final snapshot."""
    CASES[("cpu", cpu_t)] = run_case(oracle, ctxs, ("cpu", cpu_t))


def test_table_clamp_counts(oracle, ctxs):
    """Counts at table_clamp(ne) - 1, table_clamp(ne), table_clamp(ne) + 1 for a 20 000-node group (clamp 214 748): the
    tables answer up to the clamp, the scan above it; both against the oracle."""
    rng = np.random.default_rng(5)
    n = 20000
    clamp = 0xFFFFFFFF // n
    cpu = np.full(n, 64000, np.int64)
    mem = (12 << 30) + rng.integers(-1, 2, n).astype(np.int64)          # 11 or 12 executors of 2^30, at the boundary
    gpu = np.zeros(n, np.int64)
    order = rng.permutation(n).astype(np.int32)
    q = 9
    a = {"drv_cpu": np.zeros(q, np.int64), "drv_mem": np.array([0, 0, 0, 1 << 30, 1 << 30, 1 << 30, 0, 0, 0], np.int64),
         "drv_gpu": np.zeros(q, np.int64), "exe_cpu": np.full(q, 1000, np.int64),
         "exe_mem": np.array([1 << 30] * 6 + [(1 << 30) + 1] * 3, np.int64), "exe_gpu": np.zeros(q, np.int64),
         "count": np.array([clamp - 1, clamp, clamp + 1] * 3, np.int32)}
    for algo in (0, 1):
        want, _ = _closed(oracle, algo, 0, cpu, mem, gpu, order, order, a)
        assert (want[0] >= 0).sum() >= 6
        for name in ("default", "tables0"):
            ctxs[name].set_snapshot(cpu, mem, gpu, order, order)
            assert_same_results(ctxs[name].pack_batch(a, algo, 0), want, f"clamp {name} algo {algo}")


def test_coverage_matrix(oracle, ctxs):
    """Every reachable (family, class, divider kind, gpu state) cell is hit by a checked entry call.  Cases the lattice tests
    of this session did not run (or did not pass) are run here, so the matrix does not depend on which tests ran before."""
    cov = {}
    for key in [("lattice",) + c for c in LATTICE] + [("cpu", c) for c in CPU_SWITCH]:
        if key not in CASES:
            CASES[key] = run_case(oracle, ctxs, key)
        for cell, v in CASES[key].items():
            cov[cell] = cov.get(cell, 0) + v
    lines = ["family      class    kind    " + "  ".join(f"{g:>9}" for g in (IDLE, USED))]
    for fam in FAMILIES:
        for cls in m.CLASSES:
            for k in m.KINDS:
                row = [cov.get((fam, cls, k, g), 0) for g in (IDLE, USED)]
                reach = [(fam, cls, k, g) in REACHABLE for g in (IDLE, USED)]
                if any(reach) or any(row):
                    lines.append(f"{fam:11} {cls:8} {k:7} " + "  ".join(f"{v if r else '-':>9}" for v, r in zip(row, reach)))
    print("\n" + "\n".join(lines))
    missing = sorted(c for c in REACHABLE if not cov.get(c))
    assert not missing, missing
    extra = sorted(c for c in cov if c not in REACHABLE)
    assert not extra, extra


# ---------------------------------------------------------------------------------------------------------------------
# Part B: scale invariance
# ---------------------------------------------------------------------------------------------------------------------
def _scaled(a, fc, fm, fg):
    b = dict(a)
    for k, f in (("cpu", fc), ("mem", fm), ("gpu", fg)):
        for p in ("drv_", "exe_"):
            if p + k in a:
                b[p + k] = np.asarray(a[p + k], np.int64) * f
    return b


SCALES = [(3, 1000, 1), ((1 << 32) + 1, 3, 1000), (1000, 1 << 20, (1 << 32) + 1)]


@pytest.mark.parametrize("fc,fm,fg", SCALES)
def test_scale_invariance_headline(ctxs, fc, fm, fg):
    """The headline workload (10 000 nodes x 100 000 applications), algos 0, 1, 2: scaled == unscaled, bit for bit; the
    factors move requests across fast32, fast64 (none here), general and kDivSlow."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000)
    apps = synth.make_apps(100000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    a = {k: apps[k] for k in KEYS}
    a["drv_gpu"] = (np.arange(100000) % 97 == 0).astype(np.int64)      # a few gpu-bound drivers
    g = np.where(np.arange(10000) % 3 == 0, 8, 0).astype(np.int64)
    meta = m.SnapMeta(nodes["avail_cpu"] * fc, nodes["avail_mem"] * fm, g * fg)
    assert max(meta.max_avail) < m.MAX_QUANTITY
    b = _scaled(a, fc, fm, fg)
    for name in ("default", "tables0"):
        p = ctxs[name]
        for algo in (0, 1, 2):
            p.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], g, order, order)
            want = p.pack_batch(a, algo, 0)
            p.set_snapshot(nodes["avail_cpu"] * fc, nodes["avail_mem"] * fm, g * fg, order, order)
            got = p.pack_batch(b, algo, 0)
            assert_same_results(got, want, f"headline x({fc}, {fm}, {fg}) {name} algo {algo}")
            assert (want[0] >= 0).sum() > 50000


@pytest.mark.parametrize("mode", [1, 2])
def test_scale_invariance_fifo_da_50k(ctxs, mode):
    """fifo-da-50k (10 000 nodes in 16 groups, 50 000 queued drivers): decisions identical and the final snapshot scaled."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000, groups=16)
    apps = synth.make_apps(50000, groups=16, da_sweep=True, young_frac=0.05)
    eoff, eorder = synth.group_orders(nodes)
    a = {k: apps[k] for k in KEYS + ("group", "young")}
    for fc, fm, fg in SCALES[1:]:
        b = _scaled(a, fc, fm, fg)
        for name in ("default", "warp0"):
            p = ctxs[name]
            for algo in (0, 1):
                p.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
                want = p.pack_batch(a, algo, mode)
                f0 = p.get_snapshot()
                p.set_snapshot(nodes["avail_cpu"] * fc, nodes["avail_mem"] * fm, nodes["avail_gpu"] * fg, eorder, eorder, eoff, eoff)
                got = p.pack_batch(b, algo, mode)
                assert_same_results(got, want, f"fifo-da-50k x({fc}, {fm}, {fg}) {name} algo {algo} mode {mode}")
                f1 = p.get_snapshot()
                for x, y, f in zip(f1, f0, (fc, fm, fg)):
                    assert np.array_equal(x, y * f), (fc, fm, fg, name, algo, mode)


@pytest.mark.parametrize("s", [0, 10, 20])
def test_scale_invariance_wire32(gangpack, ctxs, s):
    """32-bit wire quantities with mem_shift = s on a snapshot whose memory is scaled by 2^s == the 64-bit layout unscaled."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000)
    apps = synth.make_apps(20000, gpu_variant=True)
    mib = nodes["avail_mem"] >> 20                                       # whole MiB
    order = synth.priority_order(nodes["avail_cpu"], mib)
    a = {k: apps[k] for k in KEYS}
    a["exe_mem"] = a["exe_mem"] >> 20; a["drv_mem"] = a["drv_mem"] >> 20
    a["exe_mem"][::5] += 1                                               # odd request units
    w32 = {k: np.asarray(a[k], np.int32) for k in KEYS}
    p = ctxs["default"]
    for algo in (0, 1):
        p.set_snapshot(nodes["avail_cpu"], mib, nodes["avail_gpu"], order, order)
        want = p.pack_batch(a, algo, 0)
        p.set_snapshot(nodes["avail_cpu"], mib << s, nodes["avail_gpu"], order, order)
        got = p.pack_batch(w32, algo, 0, wire=dict(quantity_bits=32, mem_shift=s, node_bits=32))
        assert_same_results(got, want, f"wire32 mem_shift {s} algo {algo}")


def _zone_inputs(rng, n, Z):
    alloc = [rng.integers(4, 97, n) * 1000, rng.integers(16, 385, n) * GI + rng.integers(0, 3, n) * (1 << 20),
             np.where(rng.random(n) < 0.3, 8, 0)]
    R_ = 3 * n
    rnode = rng.integers(0, n, R_).astype(np.int32)
    res = [rng.integers(0, 4, R_) * 1000, rng.integers(0, 16, R_) * (1 << 29), np.zeros(R_, np.int64)]
    zone = rng.integers(0, Z, n).astype(np.int32)
    return [np.asarray(x, np.int64) for x in alloc], rnode, [np.asarray(x, np.int64) for x in res], zone


@pytest.mark.parametrize("kc,km", [(1, 1 << 10), (1 << 32, 2), (1 << 16, 1 << 4)])   # cluster sums stay below 2^61
def test_scale_invariance_zones_and_efficiency(gangpack, ctxs, kc, km):
    """Zone packers, az-aware packing and the packing efficiency, with power-of-two factors on whole-core inputs (the float64
    efficiency ratios are then exactly invariant): zones, drivers, executors and efficiencies identical."""
    from k8s_spark_scheduler_b200 import native
    rng = np.random.default_rng(kc % 1000 + km)
    n, Z, q = 3000, 3, 4000
    alloc, rnode, res, zone = _zone_inputs(rng, n, Z)
    rank = rng.permutation(n).astype(np.int32)
    qa = {"drv_cpu": rng.integers(1, 3, q) * 1000, "drv_mem": rng.integers(1, 5, q) * GI, "drv_gpu": np.zeros(q, np.int64),
          "exe_cpu": rng.integers(1, 5, q) * 1000, "exe_mem": rng.integers(1, 17, q) * GI + (rng.random(q) < 0.2) * (1 << 20),
          "exe_gpu": (rng.random(q) < 0.05).astype(np.int64), "count": rng.integers(0, 40, q).astype(np.int32),
          "young": (rng.random(q) < 0.5).astype(np.uint8)}
    qa = {k: np.asarray(v, np.int64 if k not in ("count", "young") else v.dtype) for k, v in qa.items()}
    p = ctxs["default"]

    def run(fc, fm):
        al = [alloc[0] * fc, alloc[1] * fm, alloc[2]]
        rs = [res[0] * fc, res[1] * fm, res[2]]
        b = _scaled(qa, fc, fm, 1)
        out = {}
        p.prepare_cluster_zones(al, None, rnode, rs, zone, Z, rank, kind=native.LAYOUT_SINGLE_AZ)
        for algo in (0, 2):
            out[f"zones{algo}"] = p.pack_batch_zones(b, algo)
        p.prepare_cluster_zones(al, None, rnode, rs, zone, Z, rank, kind=native.LAYOUT_SINGLE_AZ)
        out["fifo_zones"] = p.pack_fifo_zones(b, 0, 1)
        out["fifo_zones_snap"] = p.get_snapshot()
        p.prepare_cluster_zones(al, None, rnode, rs, zone, Z, rank, kind=native.LAYOUT_AZ_AWARE)
        out["az"] = p.pack_batch_az_aware(b)
        out["az_fifo"] = p.pack_fifo_az_aware(b, 2)
        out["az_fifo_snap"] = p.get_snapshot()
        av, _ = p.build_availability(al, None, rnode, rs)
        d, e = p.potential_nodes(av[0], av[1], zone, Z, rank)
        p.set_snapshot(av[0], av[1], av[2], e, d)
        p.set_schedulable(*al)
        placed = p.pack_batch(b, 0, 0)
        out["eff"] = p.packing_efficiency(b, placed, 0)
        out["exceeds"] = p.exceeds_cluster_capacity(al, b, 0, zone_id=zone, n_zones=Z)
        return out

    base, sc = run(1, 1), run(kc, km)
    for key in base:
        x, y = base[key], sc[key]
        if key.endswith("_snap"):
            for u, v, f in zip(y, x, (kc, km, 1)):
                assert np.array_equal(u, v * f), key
        elif key in ("eff", "exceeds"):
            assert np.array_equal(x, y), key
        else:                                                          # zone, driver, executors, off, efficiencies
            placed = x[1] >= 0
            assert np.array_equal(x[0], y[0]), key
            assert_same_results(y[1:4], x[1:4], key)                   # ExecutorNodes of the placed applications
            assert np.array_equal(x[4][placed], y[4][placed]), key
    assert (base["zones0"][1] >= 0).sum() > q // 2 and (base["az"][1] >= 0).sum() > q // 2


# ---------------------------------------------------------------------------------------------------------------------
# Part C: mutations across a boundary on one long-lived context
# ---------------------------------------------------------------------------------------------------------------------
def test_usage_delta_lifts_the_view_shift(oracle, gangpack, ctxs):
    """Memory maximum just below 2^36 (view shift 4); a negative usage delta lifts one node to 2^36 + 2^30 (shift 5).  Then
    independent packs (algos 0, 1, 2), a zone pack, reservations that drive a gpu negative, a FIFO batch and packs again:
    after each step the long-lived context must agree with a fresh one built from its snapshot and with the oracle."""
    rng = np.random.default_rng(36)
    n = 300
    cpu = rng.integers(8, 97, n).astype(np.int64) * 1000
    mem = rng.integers(1, 63, n).astype(np.int64) << 30
    mem[0] = (1 << 36) - 1
    gpu = np.where(np.arange(n) % 4 == 0, 2, 0).astype(np.int64)
    zone_of = np.arange(n) % 2
    order = np.argsort(-mem, kind="stable").astype(np.int32)
    order = np.concatenate([order[1:2], order[:1], order[2:]]).astype(np.int32)
    eo = np.concatenate([order[zone_of[order] == z] for z in (0, 1)]).astype(np.int32)
    eoff = np.array([0, (zone_of == 0).sum(), n], np.int32)
    lifted = int(order[0])
    q = 400
    a = {"drv_cpu": rng.integers(0, 3, q) * 1000, "drv_mem": rng.integers(0, 3, q) << 30, "drv_gpu": np.zeros(q, np.int64),
         "exe_cpu": rng.choice([1000, 2000, 3], q), "exe_mem": rng.choice([1 << 30, 3 << 30, 1 << 28, (1 << 30) + 1, 1 << 34], q),
         "exe_gpu": np.zeros(q, np.int64), "count": rng.integers(1, 120, q).astype(np.int32), "group": (np.arange(q) % 2).astype(np.int32)}
    a = {k: np.asarray(v) for k, v in a.items()}
    p = ctxs["default"]
    fresh = gangpack.GangPacker()
    sched = (cpu + 4000, mem + (8 << 30), gpu + 1)
    try:
        p.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
        p.set_schedulable(*sched)
        assert m.SnapMeta(cpu, mem, gpu).shift32[1] == 4
        # the lift: mem[lifted] -> 2^36 + 2^30 (and a little cpu)
        p.apply_usage_delta([lifted], [1000], [(1 << 36) + (1 << 30) - int(mem[lifted])], [0], sign=-1)
        snap = p.get_snapshot()
        assert int(snap[1][lifted]) == (1 << 36) + (1 << 30) and m.SnapMeta(*snap).shift32[1] == 5

        def check(step):
            s = p.get_snapshot()
            fresh.set_snapshot(*s, eo, eo, eoff, eoff)
            for algo in (0, 1, 2):
                got = p.pack_batch(a, algo, 0)
                assert_same_results(got, fresh.pack_batch(a, algo, 0), f"{step} fresh algo {algo}")
                for z in (0, 1):
                    sel = np.nonzero(a["group"] == z)[0]
                    sub = {k: a[k][sel] for k in KEYS}
                    ordz = eo[eoff[z]:eoff[z + 1]]
                    want, _ = _closed(oracle, MF_ORC if algo == 2 else algo, 0, *s, ordz, ordz, sub)
                    assert_same_results(group_slices(*got, sel), want, f"{step} oracle algo {algo} zone {z}")
            return s

        check("after the lift")
        s = p.get_snapshot()
        fresh.set_snapshot(*s, eo, eo, eoff, eoff)
        fresh.set_schedulable(*sched)
        za = {k: a[k] for k in KEYS}
        zg, zf = p.pack_batch_zones(za, 0), fresh.pack_batch_zones(za, 0)
        assert np.array_equal(zg[0], zf[0]), "zone pack: zones"
        assert_same_results(zg[1:4], zf[1:4], "zone pack vs fresh")
        names = node_names(n)
        cl = oracle.Cluster(names, *s, sched=sched, zone=["zone-%d" % z for z in zone_of])
        wd, we, woff = cl.binpack_batch(2, res_aos(a["drv_cpu"], a["drv_mem"], a["drv_gpu"]),
                                        res_aos(a["exe_cpu"], a["exe_mem"], a["exe_gpu"]), a["count"], [names[i] for i in eo],
                                        [names[i] for i in eo], with_efficiencies=True, n_threads=4)
        assert_same_results(zg[1:4], (wd, we, woff), "zone pack vs the literal C")
        assert (wd >= 0).sum() > q // 2
        check("after the zone pack")
        # reservations that drive one gpu negative: a gpu driver placed on a node with no gpu
        gpu0 = int(np.nonzero(s[2][eo[:eoff[1]]] == 0)[0][0])
        r_apps = {"drv_cpu": [1000], "drv_mem": [1 << 30], "drv_gpu": [1], "exe_cpu": [1000], "exe_mem": [1 << 30], "exe_gpu": [0],
                  "count": [1]}
        p.reserve_placements(r_apps, (np.array([eo[gpu0]], np.int32), np.array([lifted], np.int32), np.array([0, 1], np.int64)))
        s = check("after the reservation")
        assert s[2].min() < 0
        # a FIFO batch on the charged snapshot, against the oracle group by group, then packs again
        young = (rng.random(q) < 0.5).astype(np.uint8)
        fresh.set_snapshot(*s, eo, eo, eoff, eoff)
        got = p.pack_batch(dict(a, young=young), 0, 1)
        assert_same_results(got, fresh.pack_batch(dict(a, young=young), 0, 1), "fifo vs fresh")
        for x, y in zip(p.get_snapshot(), fresh.get_snapshot()):
            assert np.array_equal(x, y), "fifo final snapshot vs fresh"
        avail = s
        for z in (0, 1):
            sel = np.nonzero(a["group"] == z)[0]
            sub = {k: a[k][sel] for k in KEYS}
            ordz = eo[eoff[z]:eoff[z + 1]]
            want, avail = _closed(oracle, 0, 1, *avail, ordz, ordz, sub, young[sel])
            assert_same_results(group_slices(*got, sel), want, f"fifo zone {z}")
        for x, y in zip(p.get_snapshot(), avail):
            assert np.array_equal(x, y), "fifo final snapshot"
        check("after the FIFO batch")
    finally:
        fresh.close()
