"""gp_reconcile_find_nodes_resident: the failover reconciler over the resident reservation and overhead tables.

It must return what gp_reconcile_find_nodes returns on the equivalent gp_usage_input -- reservations.to_usage_rows of the
mirror of the reservation table, and as overhead the host arrays or gp_overhead_table_query's GetOverhead -- bit for bit:
placed, every ExecutorNodes slice, the availability after the loop and the status.  Checked over random event streams
through both tables, node-table entries without an id, empty groups, no nodes, no drivers, overshoot charges that leave the
exact domain, every refusal (both tables and the held snapshot unchanged after it) and a 50 000-node x 1 000 000-slot cluster."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import native
from k8s_spark_scheduler_b200 import reservations as rv
from test_overhead_table_model import Driver as OverheadDriver, churn as overhead_churn
from test_reservation_table_model import Driver, churn

pytestmark = pytest.mark.gpu

GIB = 1 << 30
INVALID, UNREPRESENTABLE = 1, 6


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def outcome(fn):
    """(status, result): GP_OK and the result, or the refusal's status and None"""
    try:
        return 0, fn()
    except native.GangpackError as e:
        return e.status, None


def defined(r):
    """reconcile_find_nodes' result without the entries past placed[i], which are undefined"""
    if r is None:
        return None
    placed, execn, off, av = r
    slices = [execn[off[i]:off[i] + max(int(placed[i]), 0)].tolist() for i in range(len(placed))]
    return placed.tolist(), slices, off.tolist(), None if av is None else [x.tolist() for x in av]


class Nodes:
    """A node table over names n0..n{n-1}; instance group G-1 has no node, so its drivers are not placed"""

    def __init__(self, rng, n, G):
        self.names = [f"n{i}" for i in range(n)]
        self.alloc = [rng.integers(4, 33, n) * 1000, rng.integers(8, 129, n) * GIB, rng.integers(0, 5, n)]
        self.over = [rng.integers(0, 3, n) * 250, rng.integers(0, 3, n) * (1 << 28), np.zeros(n, np.int64)]
        self.group = rng.integers(0, max(G - 1, 1), n).astype(np.int32)
        self.creation = rng.integers(0, 50, n).astype(np.int64)           # ties broken by node-table index
        self.unsched = (rng.random(n) < 0.1).astype(np.uint8)
        self.ready = (rng.random(n) > 0.1).astype(np.uint8)
        self.G = G

    def apps(self, rng, q):
        return dict(exe_cpu=rng.integers(1, 9, q) * 500, exe_mem=rng.integers(1, 17, q) * (GIB // 2),
                    exe_gpu=(rng.random(q) < 0.2).astype(np.int64), count=rng.integers(0, 7, q).astype(np.int32),
                    group=rng.integers(0, self.G, q).astype(np.int32))

    def pair(self, p, rdrv, apps, present=None, overhead=None, overhead_node_id=None, want_avail=True):
        """(per-call, resident) outcomes on the nodes `present` (default all, in order)"""
        present = np.arange(len(self.names)) if present is None else np.asarray(present)
        ids = rdrv.table.node_ids([self.names[i] for i in present])
        rnode, res = rv.to_usage_rows(rdrv.mirror, ids)
        alloc = [a[present] for a in self.alloc]
        if overhead is None and overhead_node_id is None:
            overhead = [o[present] for o in self.over]
        kw = dict(unschedulable=self.unsched[present], ready=self.ready[present], want_avail=want_avail)
        a = outcome(lambda: p.reconcile_find_nodes(alloc, overhead, rnode, res, self.group[present], self.creation[present], apps,
                                                   self.G, **kw))
        b = outcome(lambda: p.reconcile_find_nodes_resident(ids, alloc, None if overhead_node_id is not None else overhead,
                                                            self.group[present], self.creation[present], apps, self.G,
                                                            overhead_node_id=overhead_node_id, **kw))
        return (a[0], defined(a[1])), (b[0], defined(b[1]))


@pytest.mark.parametrize("seed", range(4))
def test_random_streams(packer, seed):
    """after every flush of both tables: overhead from the host arrays and from the overhead table, all nodes and a subset"""
    rng = np.random.default_rng(seed)
    nodes = Nodes(rng, 48, 2 + seed)
    rdrv, odrv = Driver(), OverheadDriver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
    names = nodes.names[:40] + ["gone-0", "gone-1"]                       # slots whose node id no entry carries
    steps = zip(churn(rng, rdrv, names, 8, 2 + 3 * seed), overhead_churn(rng, odrv, 46, 8, 4))
    placed_somewhere = unplaced = 0
    for s, (d, od) in enumerate(steps):
        rdrv.table.push(packer, d)
        odrv.table.push(packer, od)
        apps = nodes.apps(rng, 30)
        present = np.sort(rng.permutation(48)[:36]) if s % 2 else None    # nodes leaving the node table
        sub = nodes.names if present is None else [nodes.names[i] for i in present]
        a, b = nodes.pair(packer, rdrv, apps, present)
        assert a == b, ("host", seed, s)
        over = odrv.table.answer(sub, packer.overhead_table_query)[0]
        a, b = nodes.pair(packer, rdrv, apps, present, overhead=over, overhead_node_id=odrv.table.node_ids(sub))
        assert a[0] == 0 and a == b, ("table", seed, s)
        placed_somewhere += sum(x > 0 for x in a[1][0])
        unplaced += sum(x == -1 for x in a[1][0])
    assert rdrv.replays >= 1 and placed_somewhere and unplaced


def test_no_nodes_and_no_drivers(packer):
    rng = np.random.default_rng(5)
    nodes = Nodes(rng, 30, 3)
    rdrv = Driver()
    for d in churn(rng, rdrv, nodes.names, 2, 5):
        rdrv.table.push(packer, d)
    apps = nodes.apps(rng, 12)
    a, b = nodes.pair(packer, rdrv, apps, present=np.zeros(0, np.int64))          # n_nodes == 0: every driver -1
    assert a == b and a[0] == 0 and a[1][0] == [-1] * 12
    none = {k: v[:0] for k, v in apps.items()}
    a, b = nodes.pair(packer, rdrv, none)                                           # q == 0 with the availability asked for
    assert a == b and a[0] == 0 and len(a[1][3][0]) == 30
    a, b = nodes.pair(packer, rdrv, none, want_avail=False)
    assert a == b and a[0] == 0
    ids = np.full(30, -1, np.int32)                                                 # no entry carries an id
    got = packer.reconcile_find_nodes_resident(ids, nodes.alloc, nodes.over, nodes.group, nodes.creation, apps, nodes.G)
    want = packer.reconcile_find_nodes(nodes.alloc, nodes.over, np.zeros(0, np.int32), (np.zeros(0, np.int64),) * 3, nodes.group,
                                       nodes.creation, apps, nodes.G)
    assert defined(got) == defined(want)


def test_overshoot_leaving_the_domain(packer):
    """each driver overshoots once more; the third charge leaves the exact domain: both forms refuse it the same way"""
    big = (1 << 60) + 7
    packer.reservation_table_reset(4, 2)
    packer.reservation_table_update(dict(slot=[0], node_id=[1], cpu_milli=[-5], mem_bytes=[0]))
    alloc = [np.array([1 << 60], np.int64), np.array([1 << 50], np.int64), np.zeros(1, np.int64)]
    group, creation = np.zeros(1, np.int32), np.ones(1, np.int64)
    for k, want in ((3, UNREPRESENTABLE), (1, 0)):
        apps = dict(exe_cpu=np.full(k, big), exe_mem=np.zeros(k, np.int64), count=np.ones(k, np.int32), group=np.zeros(k, np.int32))
        a = outcome(lambda: packer.reconcile_find_nodes(alloc, None, np.zeros(1, np.int32), ([-5], [0], [0]), group, creation, apps, 1))
        b = outcome(lambda: packer.reconcile_find_nodes_resident(np.array([1], np.int32), alloc, None, group, creation, apps, 1))
        assert (a[0], defined(a[1])) == (b[0], defined(b[1])) and a[0] == want, k


def held_state(p, names, rdrv, odrv, alloc):
    """what a refused call must leave: a following resident prepare over both tables, and the snapshot it lays out"""
    ids, oids = rdrv.table.node_ids(names), odrv.table.node_ids(names)
    r = p.prepare_cluster_groups_resident(ids, alloc, None, None, 1, overhead_node_id=oids)
    return r, p.get_snapshot()


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and np.array_equal(a, b)
    return a == b


def test_refusals_leave_both_tables_and_the_snapshot(gangpack):
    p = gangpack.GangPacker()
    try:
        rng = np.random.default_rng(17)
        nodes = Nodes(rng, 40, 3)
        apps = nodes.apps(rng, 20)
        ids = np.arange(40, dtype=np.int32)
        call = lambda node_id=ids, oid=None, **kw: outcome(lambda: p.reconcile_find_nodes_resident(
            node_id, nodes.alloc, None if oid is not None else nodes.over, kw.pop("group", nodes.group), nodes.creation,
            kw.pop("apps", apps), kw.pop("G", nodes.G), overhead_node_id=oid, **kw))[0]
        assert call() == INVALID                                                    # no reservation table
        rdrv = Driver(n_slots=64, n_node_ids=40)
        for d in churn(rng, rdrv, nodes.names, 3, 6):
            rdrv.table.push(p, d)
        assert call() == 0
        assert call(oid=ids) == INVALID                                             # overhead_node_id without an overhead table
        odrv = OverheadDriver(n_slots=64, n_node_ids=48, n_app_keys=8, n_app_ids=8, n_names=64)
        for od in overhead_churn(rng, odrv, 38, 3, 8):
            odrv.table.push(p, od)
        oids = odrv.table.node_ids(nodes.names)
        assert call(node_id=rdrv.table.node_ids(nodes.names), oid=oids) == 0
        held = held_state(p, nodes.names, rdrv, odrv, nodes.alloc)

        def with_(base, at, v):
            x = np.array(base, np.int32)
            x[at] = v
            return x
        rid = rdrv.table.node_ids(nodes.names)
        cases = [
            (INVALID, dict(group=with_(nodes.group, 3, nodes.G))),                 # per-call refusals first
            (INVALID, dict(apps=dict(apps, count=with_(apps["count"], 0, -1)))),
            (INVALID, dict(G=0)),
            (INVALID, dict(node_id=with_(rid, 5, 1 << 20))),                       # reservation-table id out of range
            (INVALID, dict(node_id=with_(rid, [5, 6], 0))),                        # given twice
            (INVALID, dict(node_id=with_(rid, 5, -2))),
            (INVALID, dict(node_id=rid, oid=with_(oids, 7, 1 << 20))),             # overhead-table id out of range
            (INVALID, dict(node_id=rid, oid=with_(oids, [7, 8], 0))),              # given twice
        ]
        for want, kw in cases:
            assert call(**kw) == want, kw
            assert same(held_state(p, nodes.names, rdrv, odrv, nodes.alloc), held), kw
        # a per-node overhead sum at 2^61: two records of 2^60 on one node of its own
        p.overhead_table_update(dict(slot=[62, 63], node_id=[47, 47], req_cpu_milli=[1 << 60, 1 << 60], req_mem_bytes=[0, 0],
                                     listed=[1, 1], app_key=[-1, -1], app_id=[-1, -1], name_id=[0, 0]))
        over_sum = with_(np.where(oids == 47, -1, oids), 11, 47)
        assert call(node_id=rid, oid=over_sum) == UNREPRESENTABLE
        p.overhead_table_update(dict(slot=[62, 63], node_id=[-1, -1], req_cpu_milli=[0, 0], req_mem_bytes=[0, 0],
                                     app_key=[-1, -1], app_id=[-1, -1], name_id=[0, 0]))
        assert same(held_state(p, nodes.names, rdrv, odrv, nodes.alloc), held)
        assert call(node_id=rid, oid=oids) == 0                                     # and the resident call leaves them too
        assert same(held_state(p, nodes.names, rdrv, odrv, nodes.alloc), held)
    finally:
        p.close()


def test_full_size_with_churn(packer):
    """50 000 nodes x 1 000 000 slots, 1 % churn, 16 instance groups, 300 stale drivers, overhead from both tables"""
    rng = np.random.default_rng(50_000)
    n, n_rows, G, q = 50_000, 1_000_000, 16, 300
    nodes = Nodes(rng, n, G + 1)
    drv = Driver(n_slots=2 * n_rows, n_node_ids=n)
    for r in range(n_rows // 20):
        drv.table.rr_set(("ns", f"app-{r}"), {f"e{j}": (nodes.names[rng.integers(n)], int(rng.integers(1, 5)) * 250,
                                                         int(rng.integers(1, 9)) << 28, 0) for j in range(20)})
    drv.table.push(packer, drv.step())
    keys = list(drv.table.rrs)
    for s in range(2):
        for k in rng.choice(len(keys), len(keys) // 100, replace=False):           # 1 % of the rows rewritten
            drv.table.rr_set(keys[k], {e: (nodes.names[rng.integers(n)],) + r[1:] for e, r in drv.table.rrs[keys[k]].items()})
        d = drv.step()
        assert d["reset"] is None
        drv.table.push(packer, d)
        apps = nodes.apps(rng, q)
        apps["count"] = rng.integers(0, 40, q).astype(np.int32)
        a, b = nodes.pair(packer, drv, apps)
        assert a[0] == 0 and a == b, s
        assert any(x > 0 for x in a[1][0]) and -1 in a[1][0]
