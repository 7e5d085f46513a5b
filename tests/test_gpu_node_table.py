"""The resident node table (gp_node_table_reset / _update) and the node-table Predicate entries
(gp_prepare_cluster_groups_node_table, gp_prepare_cluster_zones_groups_node_table, gp_reschedule_from_reservations_node_table).

Each node-table entry must give what its *_resident entry gives on the columns decoded from the numpy mirrors of the node
and label tables (nodes.NodeMirror.to_columns, nodes.label_columns) -- bit for bit: orders, offsets, counts, undefined ties,
the zone layout, get_snapshot, node_out and ambiguous -- after every flush of seeded churn over node, label, reservation and
overhead events.  Every refusal is checked once: a refused delta leaves the table as it was (the next call's identity shows
it), and a refused call leaves the context as it was."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import affinity, native, nodes
from test_overhead_table_model import Driver as OverheadDriver, churn as overhead_churn
from test_reservation_table_model import Driver as ReservationDriver, churn as reservation_churn

pytestmark = pytest.mark.gpu

INVALID, UNREPRESENTABLE = 1, 6
ZONES = ["z0", "z1", "z2"]
GROUPS = ["g0", "g1", "g2"]
PRIORITY = ["p2", "p0", "p1"]


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def outcome(fn):
    try:
        return 0, fn()
    except native.GangpackError as e:
        return e.status, None


def same(a, b, label):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), label
        for k in a:
            same(a[k], b[k], (label, k))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), label
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, (label, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and np.array_equal(a, b), label
    else:
        assert a == b, label


class World:
    """n node names n0.. with labels, allocatable and flags churned in the node and label tables, plus reservation and
    overhead churn over the same names"""

    def __init__(self, seed, n, key_bits=62):
        self.rng = np.random.default_rng(seed)
        self.n = n
        self.labels = affinity.LabelTable(n_node_ids=8, n_keys=8, n_values=8)
        self.table = nodes.NodeTable(self.labels, n_node_ids=8, key_bits=key_bits)
        self.rdrv = ReservationDriver()
        self.odrv = OverheadDriver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
        self.rstream = reservation_churn(self.rng, self.rdrv, [f"n{i}" for i in range(n + 2)], 10 ** 9, max(2, n // 100))
        self.ostream = overhead_churn(self.rng, self.odrv, n, 10 ** 9, max(2, n // 100))
        self.order = self.rng.permutation(n)            # node names are added in a random order: inserts before, between, after
        self.added = 0

    def node_event(self, name):
        r = self.rng
        lab = {}
        if r.random() < 0.85:
            lab[nodes.ZONE_LABEL] = ZONES[r.integers(len(ZONES))]
        if r.random() < 0.8:
            lab["instance-group"] = (GROUPS + ["gx"])[r.integers(len(GROUPS) + 1)]
        if r.random() < 0.6:
            lab["priority"] = (PRIORITY + ["px"])[r.integers(len(PRIORITY) + 1)]
        self.labels.set_node(name, lab)
        # few distinct (cpu, mem): equal (mem, cpu) with a different gpu makes undefined ties
        alloc = (int(r.integers(2, 5)) * 16000, int(r.integers(2, 5)) * (64 << 30), int(r.integers(0, 3)))
        self.table.set_node(name, alloc, r.random() < 0.05, r.random() < 0.95)

    def churn(self, k):
        r = self.rng
        for _ in range(k):
            live = list(self.table.nodes)
            op = r.random()
            if self.added < self.n and (op < 0.5 or not live):
                self.node_event(f"n{self.order[self.added]}")
                self.added += 1
            elif op < 0.7 and len(live) > 4:
                name = live[r.integers(len(live))]
                self.table.delete_node(name)
                self.labels.delete_node(name)
            else:
                self.node_event(live[r.integers(len(live))]) if live else None

    def flush(self, p):
        self.labels.flush(p)
        self.table.flush(p)
        self.rdrv.table.push(p, next(self.rstream))
        self.odrv.table.push(p, next(self.ostream))

    def listed(self, subset=True):
        names = list(self.table.nodes)
        if subset and len(names) > 8:
            names = [names[i] for i in self.rng.permutation(len(names))[: len(names) - len(names) // 8]]
        return names

    def nodes_dict(self, names, priorities=True, zone=True, candidates=True):
        args = nodes.label_args(self.labels, zones=ZONES if zone else None, zone_label=nodes.ZONE_LABEL if zone else "no-such-label",
                                instance_group_label="instance-group", instance_groups=GROUPS,
                                driver_priority=("priority", PRIORITY) if priorities else None,
                                executor_priority=("priority", PRIORITY[::-1]) if priorities else None)
        cand = (self.rng.random(len(names)) < 0.9).astype(np.uint8) if candidates else None
        return dict(node_table_id=self.table.node_ids(names), reservation_id=self.rdrv.table.node_ids(names),
                    overhead_node_id=self.odrv.table.node_ids(names), is_driver_candidate=cand, **args)

    def decoded(self, nd):
        cols = self.table.mirror.to_columns(nd["node_table_id"])
        lab = nodes.label_columns(self.labels.mirror, **nd)
        return cols, lab


def check(p, w, label, names=None, priorities=True, zone=True, ig_from_labels=True):
    names = w.listed() if names is None else names
    nd = w.nodes_dict(names, priorities, zone)
    cols, lab = w.decoded(nd)
    G = len(GROUPS)
    n_zones = nd["n_zones"]
    sa = (lab["zone_id"], n_zones, cols["name_rank"], nd["is_driver_candidate"], cols["unschedulable"], cols["ready"],
          lab["driver_label_rank"], lab["executor_label_rank"])
    ig = lab["instance_group"]
    rid, oid = nd["reservation_id"], nd["overhead_node_id"]

    def pair(resident, node_table):
        a = outcome(resident)
        a = (a, p.get_snapshot() if a[0] == 0 else None)
        b = outcome(node_table)
        b = (b, p.get_snapshot() if b[0] == 0 else None)
        same(a, b, label)
        assert a[0][0] == 0, (label, a[0][0])
        return a

    zone_out, ig_out = np.full(len(names), -9, np.int32), np.full(len(names), -9, np.int32)
    ndo = dict(nd, zone_id_out=zone_out, instance_group_out=ig_out)
    igx = None if ig_from_labels else ig
    pair(lambda: p.prepare_cluster_groups_resident(rid, cols["alloc"], None, ig, G, *sa, overhead_node_id=oid),
         lambda: p.prepare_cluster_groups_node_table(ndo, igx, G))
    assert np.array_equal(zone_out, lab["zone_id"] if lab["zone_id"] is not None else np.zeros(len(names), np.int32))
    assert np.array_equal(ig_out, ig)
    for kind in (native.LAYOUT_AZ_AWARE, native.LAYOUT_SINGLE_AZ):
        pair(lambda: p.prepare_cluster_zones_groups_resident(rid, cols["alloc"], None, ig, G, *sa, kind=kind, overhead_node_id=oid),
             lambda: p.prepare_cluster_zones_groups_node_table(nd, igx, G, kind=kind))
    q = 24
    r = w.rng
    exe = (r.integers(1, 9, q) * 2000, r.integers(1, 17, q) * (1 << 30), (r.integers(0, 3, q) == 0).astype(np.int64))
    hosting = [list(r.choice(len(names), r.integers(0, 3), replace=False)) for _ in range(q)]
    rk = dict(zone_id=sa[0], n_zones=n_zones, name_rank=sa[2], unschedulable=sa[4], ready=sa[5], executor_label_rank=sa[7])
    for mf in (False, True):
        a = outcome(lambda: p.reschedule_from_reservations_resident(rid, cols["alloc"], None, exe, min_frag=mf, hosting=hosting, **rk,
                                                                    overhead_node_id=oid))
        b = outcome(lambda: p.reschedule_from_reservations_node_table(nd, exe, min_frag=mf, hosting=hosting))
        same(a, b, (label, "reschedule", mf))


@pytest.mark.parametrize("seed,n,key_bits", [(1, 200, 62), (2, 300, 9), (3, 120, 62)])
def test_churn_identity(packer, seed, n, key_bits):
    w = World(seed, n, key_bits)
    ties = 0
    for s in range(12):
        w.churn(n // 3 if s == 0 else max(4, n // 20))
        w.flush(packer)
        check(packer, w, (seed, s), priorities=s % 3 != 0, zone=s % 4 != 1, ig_from_labels=s % 2 == 0)
        o = packer.prepare_cluster_groups_node_table(w.nodes_dict(w.listed(False)), None, len(GROUPS))
        ties += o["undefined_ties"]
    assert ties > 0                                    # equal (mem, cpu) with a different gpu was met
    if key_bits < 62:
        assert w.table.relabels > 0


def test_churn_identity_10000_nodes(packer):
    w = World(11, 10000)
    w.churn(10000)
    w.flush(packer)
    for s in range(3):
        check(packer, w, ("10k", s))
        w.churn(100)                                   # 1 % churn
        w.flush(packer)
    check(packer, w, ("10k", "last"), names=w.listed(False))


def status_of(fn):
    return outcome(fn)[0]


def test_refused_deltas_leave_the_table(packer):
    w = World(21, 60)
    w.churn(60)
    w.flush(packer)
    check(packer, w, "before")
    a, b = list(w.table.nodes)[:2]
    ia, ib = (int(x) for x in w.table.node_ids([a, b]))
    row = dict(present=[1], alloc_cpu_milli=[1], alloc_mem_bytes=[1], alloc_gpu=[0], unschedulable=[0], ready=[1])
    two = {k: v * 2 for k, v in row.items()}
    bad = [
        (INVALID, dict(row, node_id=[w.table.size["n_node_ids"]], name_key=[5])),                      # id out of range
        (INVALID, dict(row, node_id=[-1], name_key=[5])),
        (INVALID, dict(two, node_id=[ia, ia], name_key=[w.table.name_key(a), w.table.name_key(a)])),      # id given twice
        (INVALID, dict(row, node_id=[ia], name_key=[w.table.name_key(b)])),                              # duplicate name_key
        (INVALID, dict(row, node_id=[ia], name_key=[(1 << 63) - 1])),
        (UNREPRESENTABLE, dict(row, node_id=[ia], name_key=[w.table.name_key(a)], alloc_cpu_milli=[1 << 61])),
        (UNREPRESENTABLE, dict(row, node_id=[ib], name_key=[w.table.name_key(b)], alloc_mem_bytes=[-(1 << 61)])),
        (INVALID, dict(row, node_id=[ia], name_key=None)),                                               # missing array
    ]
    for want, d in bad:
        assert status_of(lambda: packer.node_table_update(d)) == want, d
        check(packer, w, ("after refusal", want))
    # a swap of two keys in one delta is accepted: uniqueness is of the table after the delta
    d = dict(two, node_id=[ia, ib], name_key=[w.table.name_key(b), w.table.name_key(a)])
    packer.node_table_update(d)
    w.table.replay()
    w.table.flush(packer)
    check(packer, w, "after replay")


def test_no_label_table_is_refused(gangpack):
    p = gangpack.GangPacker()
    try:
        p.node_table_reset(n_node_ids=4)
        one = dict(node_table_id=[0], reservation_id=[-1], overhead_node_id=[-1])
        assert status_of(lambda: p.prepare_cluster_groups_node_table(one, None, 1)) == INVALID
    finally:
        p.close()


def test_refused_calls_leave_the_context(gangpack):
    p = gangpack.GangPacker()
    try:
        w = World(31, 40)
        w.churn(40)
        names = w.listed(False)
        nd = w.nodes_dict(names)
        assert status_of(lambda: p.prepare_cluster_groups_node_table(nd, None, 3)) == INVALID      # no node table yet
        w.flush(p)
        # a node listed twice, before any call has sorted this many nodes: the refused call's sort still sees unique name ranks
        dup0 = nd["node_table_id"].copy()
        dup0[1] = dup0[0]
        assert status_of(lambda: p.prepare_cluster_groups_node_table(dict(nd, node_table_id=dup0), None, 3)) == INVALID
        p.node_table_reset(n_node_ids=0)
        assert status_of(lambda: p.prepare_cluster_groups_node_table(nd, None, 3)) == INVALID      # ids out of range now
        w.table.replay()
        w.table.flush(p)
        p.prepare_cluster_groups_node_table(nd, None, 3)
        snap = p.get_snapshot()
        gone = w.table.node_ids(names).copy()
        dup = gone.copy()
        dup[1] = dup[0]
        absent = gone.copy()
        absent[0] = int(max(w.table._name_at)) + 1 if int(max(w.table._name_at)) + 1 < w.table.size["n_node_ids"] else -5
        has_zone = nodes.label_columns(w.labels.mirror, **nd)
        carried = [z for z in np.unique(has_zone["zone_id"]) if z != nd["zone_missing"]]
        unlisted = nd["zone_value"].copy()
        unlisted[carried[0]] = -99                                  # a value some node carries, not listed; "default" kept
        cases = [
            dict(nd, zone_value=unlisted),
            dict(nd, node_table_id=dup),
            dict(nd, node_table_id=absent),
            dict(nd, node_table_id=np.where(gone == gone[0], w.table.size["n_node_ids"] + 3, gone).astype(np.int32)),
            dict(nd, zone_value=nd["zone_value"][:-1].copy(), n_zones=nd["n_zones"] - 1, zone_missing=-1),   # "default" gone
            dict(nd, zone_value=np.concatenate([nd["zone_value"][:1], nd["zone_value"][:1], nd["zone_value"][2:]]).astype(np.int32)),
            dict(nd, zone_missing=nd["n_zones"]),
            dict(nd, overhead_node_id=None),
        ]
        assert (has_zone["zone_id"] == nd["zone_missing"]).any()      # some node lacks the zone label
        for k, bad in enumerate(cases):
            for call in (lambda: p.prepare_cluster_groups_node_table(bad, None, 3),
                         lambda: p.prepare_cluster_zones_groups_node_table(bad, None, 3),
                         lambda: p.reschedule_from_reservations_node_table(bad, ([1000], [1 << 30]))):
                assert status_of(call) == INVALID, k
                same(p.get_snapshot(), snap, ("refused call", k))
        p.label_table_reset(n_node_ids=0, max_labels=0, n_keys=0, n_values=0)
        p.node_table_reset(n_node_ids=4)
        p.node_table_update(dict(node_id=[0], present=[1], alloc_cpu_milli=[1], alloc_mem_bytes=[1], unschedulable=[0], ready=[1],
                                 name_key=[7]))
        one = dict(node_table_id=[0], reservation_id=[-1], overhead_node_id=[-1])
        p.prepare_cluster_groups_node_table(one, None, 1)          # a node past the label table's rows has no labels
    finally:
        p.close()
