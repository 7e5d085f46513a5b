"""The unschedulable-pod marker's sweep from the driver table (gp_exceeds_cluster_capacity_driver_table) and the table's
affinity column.

After every flush of seeded node, label, reservation, overhead and pending-driver churn, the sweep must give, bit for bit,
what today's recipe gives on the same rows: the stale drivers restated per call by drivers.DriverMirror.stale, the drivers
outside the model set aside, and gp_exceeds_cluster_capacity_affinity_node_table over the caller's programs plus one that
matches every node -- order, exceeds, outcome and status, for every packer.  The refusals (capacity, then an affinity id
out of range) leave the driver table as it was, and the FIFO entries give the same results whether or not the affinity
column is written."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import drivers, native, nodes
from test_gpu_driver_table import snapshot
from test_gpu_node_table import GROUPS, ZONES, World, outcome, same

pytestmark = pytest.mark.gpu

INVALID, CAPACITY = 1, 5
SEC = 10 ** 9
PACKERS = range(5)
SCHEDULERS = ["spark-scheduler", "other"]
IG = "instance-group"
# required affinities of the pending drivers: None (-1, every node), selectors, terms, one that parses to an error on every
# node it reaches (Gt with a value that is not an integer) and two that match nothing
AFFS = [None,
        {"nodeSelector": {IG: "g0"}, "required": None},
        {"nodeSelector": None, "required": [{"matchExpressions": [(IG, "In", ["g1", "g2"])]}]},
        {"nodeSelector": None, "required": [{"matchExpressions": [(nodes.ZONE_LABEL, "NotIn", ["z1"])]}]},
        {"nodeSelector": {nodes.ZONE_LABEL: "z2"}, "required": [{"matchExpressions": [("priority", "Exists", [])]}]},
        {"nodeSelector": None, "required": [{"matchExpressions": [("priority", "Gt", ["x"])]}]},
        {"nodeSelector": None, "required": [{"matchExpressions": [(IG, "DoesNotExist", [])]}]},
        {"nodeSelector": {IG: "nope"}, "required": None},
        {"nodeSelector": None, "required": [{"matchExpressions": [(IG, "In", ["g2"])]},
                                            {"matchExpressions": [(nodes.ZONE_LABEL, "In", ["z0"])]}]}]
TIMEOUT, NOW = 1_000 * SEC, 2_000 * SEC


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


class Pending:
    """A seeded stream of pending-driver events over a DriverTable: adds, updates, deletes, unparseable annotations, and
    drivers outside the capacity check's model (inexact, a negative quantity or count)"""

    def __init__(self, rng, affs=AFFS, odd=0.03):
        self.rng = rng
        self.table = drivers.DriverTable(n_slots=4, n_groups=1, n_schedulers=1)
        self.affs, self.odd = affs, odd
        self.n = 0

    def resources(self):
        r = self.rng
        res = {"drv": [int(r.integers(1, 5)) * 1000, int(r.integers(1, 9)) << 30, 0],
               "exe": [int(r.integers(1, 17)) * 1000, int(r.integers(1, 33)) << 30, int(r.random() < 0.2)],
               "min": int(r.integers(0, 60))}
        exact = True
        u = r.random()
        if u < self.odd:
            exact, res["exe"][1] = False, 1 << 62
        elif u < 2 * self.odd:
            res["drv"][0] = -1000
        elif u < 3 * self.odd:
            res["min"] = -1
        return res, exact

    def set(self, uid, creation=None, scheduler=None, aff="?"):
        r = self.rng
        creation = int(r.integers(0, 2_000)) * SEC if creation is None else creation
        scheduler = SCHEDULERS[int(r.random() < 0.15)] if scheduler is None else scheduler
        aff = self.affs[r.integers(len(self.affs))] if aff == "?" else aff
        res, exact = self.resources()
        group = GROUPS[r.integers(len(GROUPS))] if r.random() < 0.9 else None
        self.table.set_driver(uid, creation, scheduler, group, res, exact, affinity=aff)

    def add(self, k=1, **kw):
        for _ in range(k):
            self.n += 1
            self.set(f"d{self.n}", **kw)
        return f"d{self.n}"

    def churn(self, k):
        r = self.rng
        for _ in range(k):
            live = list(self.table.rows)
            op = r.random()
            if op < 0.5 or len(live) < 4:
                self.add()
            elif op < 0.75:
                self.table.delete_driver(live[r.integers(len(live))])           # bound, deleted or terminating
            elif op < 0.8:
                self.table.set_driver(live[r.integers(len(live))], 0, "x", None, None)   # annotations no longer parse
            else:
                self.set(live[r.integers(len(live))])


def per_call(p, w, nd, names, t, scheduler, timeout, now, pk):
    """today's recipe: the stale rows restated per call, the ones outside the model set aside, and the affinity node-table
    entry over the interned programs plus one that matches every node"""
    progs = t.affinity_programs()
    enc = w.labels.encode_affinities(progs + [drivers.MATCH_ALL], names)
    slots, apps, outside = t.mirror.stale(scheduler, timeout, now, n_aff=len(progs))
    keep = ~outside
    st, r = outcome(lambda: p.exceeds_cluster_capacity_affinity_node_table(nd, enc, {k: v[keep] for k, v in apps.items()}, pk))
    if st:
        return st, None
    exceeds, oc = np.zeros(len(slots), np.uint8), np.full(len(slots), 2, np.uint8)
    exceeds[keep], oc[keep] = r[0], r[1]
    return 0, dict(stale_slot=slots, exceeds=exceeds, outcome=oc)


def sweep(p, w, nd, names, t, scheduler, timeout, now, pk, **kw):
    enc = w.labels.encode_affinities(t.affinity_programs(), names)
    return outcome(lambda: p.exceeds_cluster_capacity_driver_table(nd, enc, scheduler, timeout, now, pk, **kw))


def check(p, w, d, label, scheduler="spark-scheduler", timeout=TIMEOUT, now=NOW, packers=PACKERS, names=None):
    names = w.listed() if names is None else names
    nd = w.nodes_dict(names, priorities=False)
    t = d.table
    sid = t.scheduler_id(scheduler) if isinstance(scheduler, str) else scheduler
    got = None
    for pk in packers:
        got = sweep(p, w, nd, names, t, sid, timeout, now, pk)
        same(got, per_call(p, w, nd, names, t, sid, timeout, now, pk), (label, pk))
        assert got[0] == 0, (label, pk, got[0])
    return got[1]


def world(seed, n_nodes, n_drivers, **kw):
    w = World(seed, n_nodes)
    w.churn(n_nodes + n_nodes // 4)
    d = Pending(w.rng, **kw)
    d.add(n_drivers)
    return w, d


def flush(p, w, d):
    w.flush(p)
    d.table.flush(p)


@pytest.mark.parametrize("seed,n_nodes,n_drivers", [(1, 150, 300), (2, 60, 40)])
def test_churned_sweeps_match_the_per_call_recipe(packer, seed, n_nodes, n_drivers):
    w, d = world(seed, n_nodes, n_drivers)
    seen = np.zeros(3, bool)
    for step in range(6):
        if step:
            w.churn(max(4, n_nodes // 20))
            d.churn(max(4, n_drivers // 10))
        flush(packer, w, d)
        got = check(packer, w, d, ("churn", seed, step))
        seen |= [np.any(got["outcome"] == k) for k in range(3)]
    assert seen.all(), seen                 # answered, affinity-error and outside-model rows all met


def test_10000_nodes_20000_drivers(packer):
    w, d = world(7, 10_000, 20_000)
    for step in range(2):
        if step:
            w.churn(100)
            d.churn(200)
        flush(packer, w, d)
        got = check(packer, w, d, ("large", step))
        assert 5_000 < len(got["stale_slot"]) < 15_000


def test_cases(packer, gangpack):
    w, d = world(11, 80, 120)
    flush(packer, w, d)
    # no stale driver; a scheduler no driver has carried (-1); every driver stale
    assert len(check(packer, w, d, "none", now=0)["stale_slot"]) == 0
    assert len(check(packer, w, d, "no scheduler", scheduler=-1)["stale_slot"]) == 0
    got = check(packer, w, d, "all", timeout=0, now=10 ** 18)
    t = d.table
    assert len(got["stale_slot"]) == int(np.sum(t.mirror.present & (t.mirror.scheduler == t.scheduler_id("spark-scheduler"))))
    # only -1 affinities, and no listed node at all (a world of its own: its own context)
    p2 = gangpack.GangPacker()
    try:
        w2, d2 = world(12, 40, 60, affs=[None])
        flush(p2, w2, d2)
        assert (check(p2, w2, d2, "-1 only")["outcome"] != 1).all()
        check(p2, w2, d2, "no nodes", names=[])
    finally:
        p2.close()
    # creation + timeout == now is not stale, one nanosecond earlier it is; int64-extreme creation and timeout
    lo, hi = -(1 << 63), (1 << 63) - 1
    for uid, cre in (("edge", NOW - TIMEOUT), ("past", NOW - TIMEOUT - 1), ("max", hi), ("min", lo)):
        d.set(uid, creation=cre, scheduler="spark-scheduler", aff=None)
    flush(packer, w, d)
    slots = check(packer, w, d, "edge")["stale_slot"].tolist()
    assert t.slot_of("past") in slots and t.slot_of("min") in slots and t.slot_of("edge") not in slots
    assert t.slot_of("max") not in slots
    # where the sum leaves int64: max + 1 is not below max, min - 1 is below min
    slots = check(packer, w, d, "above int64", timeout=1, now=hi)["stale_slot"].tolist()
    assert slots[0] == t.slot_of("min") and t.slot_of("max") not in slots and len(slots) > 100
    assert check(packer, w, d, "below int64", timeout=-1, now=lo)["stale_slot"].tolist() == [t.slot_of("min")]


def fifo(p, d, snap, now):
    t = d.table
    p.set_snapshot(*snap)
    q = dict(requesting_slot=-1, scheduler=t.scheduler_id("spark-scheduler"), snapshot_group=t.snapshot_groups({g: i for i, g in enumerate(GROUPS)}),
             enforce_after_ns=t.group_ages(30 * SEC), now=now, n_slots=t.size["n_slots"])
    return p.pack_fifo_driver_table(q, native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE)


def test_refusals_leave_the_table(packer):
    w, d = world(21, 100, 200, odd=0)          # every driver exact: the FIFO drain below refuses inexact ones
    flush(packer, w, d)
    t = d.table
    names = w.listed()
    nd = w.nodes_dict(names, priorities=False)
    sid = t.scheduler_id("spark-scheduler")
    snap = snapshot(np.random.default_rng(21), 64, len(GROUPS))
    before = fifo(packer, d, snap, NOW)
    want = per_call(packer, w, nd, names, t, sid, TIMEOUT, NOW, 3)
    n = len(want[1]["stale_slot"])
    assert n > 2
    # capacity: refused with the size needed, then the retry answers
    assert sweep(packer, w, nd, names, t, sid, TIMEOUT, NOW, 3, cap=n - 1, retry=False)[0] == CAPACITY
    same(sweep(packer, w, nd, names, t, sid, TIMEOUT, NOW, 3, cap=1), want, "retry")
    same(sweep(packer, w, nd, names, t, sid, TIMEOUT, NOW, 3, cap=n), want, "exact cap")
    # an affinity id outside [-1, n_aff): fewer programs than the table's ids
    progs = t.affinity_programs()
    stale_ids = t.mirror.affinity[want[1]["stale_slot"]]
    short = w.labels.encode_affinities(progs[:int(stale_ids.max())], names)
    st, _ = outcome(lambda: packer.exceeds_cluster_capacity_driver_table(nd, short, sid, TIMEOUT, NOW, 3))
    assert st == INVALID
    # capacity is read after the affinity check: both wrong -> INVALID
    st, _ = outcome(lambda: packer.exceeds_cluster_capacity_driver_table(nd, short, sid, TIMEOUT, NOW, 3, cap=0, retry=False))
    assert st == INVALID
    same(fifo(packer, d, snap, NOW), before, "fifo after refusals")
    same(sweep(packer, w, nd, names, t, sid, TIMEOUT, NOW, 3), want, "sweep after refusals")
    # the FIFO entries ignore the affinity column: a replay without it (NULL: -1 everywhere) packs the same
    t.replay()
    dl = t.delta()
    dl.pop("affinity")
    t.push(packer, dl)
    same(fifo(packer, d, snap, NOW), before, "fifo without affinity")
    t.replay()
    t.flush(packer)
    same(sweep(packer, w, nd, names, t, sid, TIMEOUT, NOW, 3), want, "sweep after replay")


def test_no_driver_table_is_refused(gangpack):
    p = gangpack.GangPacker()
    try:
        w, d = world(31, 20, 10)
        w.flush(p)
        names = w.listed()
        nd = w.nodes_dict(names, priorities=False)
        enc = w.labels.encode_affinities(d.table.affinity_programs(), names)
        with pytest.raises(native.GangpackError, match="no driver table") as e:
            p.exceeds_cluster_capacity_driver_table(nd, enc, 0, TIMEOUT, NOW, 0)
        assert e.value.status == INVALID
    finally:
        p.close()
