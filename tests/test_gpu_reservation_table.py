"""The resident reservation table (gp_reservation_table_reset / _update) and the resident Predicate front ends
(gp_prepare_cluster_groups_resident, gp_prepare_cluster_zones_groups_resident, gp_reschedule_from_reservations_resident).

Each resident entry must give what its per-call entry gives on the equivalent gp_usage_input -- reservations.to_usage_rows
of the numpy mirror of the table, and as overhead the host arrays or gp_overhead_table_query's output -- bit for bit: orders,
counts, undefined ties, layout arrays, get_snapshot and a following FIFO drain; node_out and ambiguous.  Checked over random
event streams, overhead from the resident overhead table, both benchmark sizes with 1 % churn, every refusal of an update
(the table unchanged after it) and of a resident entry (the held snapshot intact after it), sums at 2^61 - 1 and 2^61, and
the table's independence from everything else of the context."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import native
from k8s_spark_scheduler_b200 import reservations as rv
from helpers import random_apps
from test_gpu_prepare_zones import sort_args
from test_gpu_prepare_zones_groups import groups_case
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


def fifo_apps(rng, G, q=60):
    apps = random_apps(rng, q, gpus=True)
    apps["group"] = rng.integers(0, G, q).astype(np.int32)
    return apps


class Case:
    """groups_case's node table, some of whose node names the reservations also use; reservation rows from the table"""

    def __init__(self, seed, n=240, G=3, Z=4):
        self.c = groups_case(seed, n, G, Z)
        self.names = list(self.c["names"])
        self.G = G
        self.rng = np.random.default_rng(seed)

    def call_rows(self, drv, present):
        return rv.to_usage_rows(drv.mirror, drv.table.node_ids([self.names[i] for i in present]))

    def check(self, p, drv, label, overhead=None, overhead_node_id=None, ig=True, present=None):
        """every resident entry == its per-call entry on the mirror's rows, context afterwards included"""
        c = self.c
        present = np.arange(len(self.names)) if present is None else present
        ids = drv.table.node_ids([self.names[i] for i in present])
        rnode, res = self.call_rows(drv, present)
        alloc = [a[present] for a in c["alloc"]]
        if overhead is None and overhead_node_id is None:
            overhead = [o[present] for o in c["over"]]
        sa = sub_sort(c, present)
        igs = c["ig"][present] if ig else None
        apps = fifo_apps(self.rng, self.G)
        oid = dict(overhead_node_id=overhead_node_id)

        def pair(call, resident, after):
            a = outcome(call)
            a = (a, after() if a[0] == 0 else None)
            b = outcome(resident)
            b = (b, after() if b[0] == 0 else None)
            same(a, b, label)
            return a

        after_groups = lambda: (p.get_snapshot(), p.pack_batch(apps, 0, native.MODE_FIFO_EXACT))
        pair(lambda: p.prepare_cluster_groups(alloc, overhead, rnode, res, igs, self.G, *sa),
             lambda: p.prepare_cluster_groups_resident(ids, alloc, None if overhead_node_id is not None else overhead, igs, self.G, *sa,
                                                       **oid), after_groups)
        after_zones = lambda: (p.get_snapshot(), p.pack_fifo_zones_groups(apps, native.BP_AZ_AWARE_TIGHTLY_PACK, 1))
        pair(lambda: p.prepare_cluster_zones_groups(alloc, overhead, rnode, res, igs, self.G, *sa),
             lambda: p.prepare_cluster_zones_groups_resident(ids, alloc, None if overhead_node_id is not None else overhead, igs, self.G,
                                                             *sa, **oid), after_zones)
        q = 40
        exe = (self.rng.integers(1, 9, q) * 250, self.rng.integers(1, 17, q) * (1 << 28), (self.rng.integers(0, 3, q) == 0).astype(np.int64))
        hosting = [list(self.rng.choice(len(present), self.rng.integers(0, 3), replace=False)) for _ in range(q)]
        rk = dict(zone_id=sa[0], n_zones=sa[1], name_rank=sa[2], unschedulable=sa[4], ready=sa[5], executor_label_rank=sa[7])
        for mf in (False, True):
            pair(lambda: p.reschedule_from_reservations(alloc, overhead, rnode, res, exe, min_frag=mf, hosting=hosting, **rk),
                 lambda: p.reschedule_from_reservations_resident(ids, alloc, None if overhead_node_id is not None else overhead, exe,
                                                                 min_frag=mf, hosting=hosting, **rk, **oid),
                 lambda: None)


def sub_sort(c, present):
    """sort_args of the node table restricted to `present` (in that order), name ranks renumbered"""
    args = list(sort_args(c))
    pick = lambda x: None if x is None else np.asarray(x)[present]
    rank = np.empty(len(present), np.int32)
    rank[np.argsort(np.asarray(c["rank"])[present], kind="stable")] = np.arange(len(present))
    return (pick(args[0]), args[1], rank, pick(args[3]), pick(args[4]), pick(args[5]), pick(args[6]), pick(args[7]))


def stream(case, drv, rng, steps, per_step):
    """churn over the case's node names and a few names of nodes that are not in the node table"""
    return churn(rng, drv, case.names[: 40] + ["gone-0", "gone-1"], steps, per_step)


@pytest.mark.parametrize("seed", range(4))
def test_random_streams_equivalence(packer, seed):
    case = Case(2100 + seed, G=1 + seed % 3)
    rng = np.random.default_rng(seed)
    drv = Driver()
    for s, d in enumerate(stream(case, drv, rng, steps=8, per_step=1 + 3 * seed)):
        drv.table.push(packer, d)
        present = rng.permutation(len(case.names))[: len(case.names) - 20] if s % 2 else None   # nodes leaving the table
        case.check(packer, drv, (seed, s), ig=seed != 3, present=present)
    assert drv.replays >= 2


def test_overhead_from_the_overhead_table(packer):
    """overhead_node_id: GetOverhead from the resident overhead table == the per-call entries given its query's output"""
    rng = np.random.default_rng(7)
    case = Case(2200, n=8, G=2, Z=2)
    case.names = [f"n{i}" for i in range(8)]                    # the overhead stream's node names
    odrv = OverheadDriver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
    drv = Driver()
    for s, (od, d) in enumerate(zip(overhead_churn(rng, odrv, 6, steps=10, per_step=3), stream(case, drv, rng, 10, 2))):
        odrv.table.push(packer, od)
        drv.table.push(packer, d)
        oids = odrv.table.node_ids(case.names)
        over = odrv.table.answer(case.names, packer.overhead_table_query)[0]
        case.check(packer, drv, ("host", s), overhead=over)                 # the query's output as host arrays on both sides
        case.check(packer, drv, ("table", s), overhead=over, overhead_node_id=oids)   # resident: from the overhead table


def cluster_rows(rng, table, nodes, n_rows, per_rr=21):
    for r in range(n_rows // per_rr):
        table.rr_set(("ns", f"app-{r}"), {f"e{j}": (nodes[rng.integers(len(nodes))], int(rng.integers(1, 9)) * 500,
                                                      int(rng.integers(1, 17)) << 28, int(rng.integers(0, 8) == 0))
                                           for j in range(per_rr)})


@pytest.mark.parametrize("n_nodes,n_rows", [(10_000, 100_000), (50_000, 1_000_000)])
def test_full_size_with_churn(packer, n_nodes, n_rows):
    rng = np.random.default_rng(n_nodes)
    names = [f"node-{i}" for i in range(n_nodes)]
    drv = Driver(n_slots=2 * n_rows, n_node_ids=n_nodes)
    cluster_rows(rng, drv.table, names, n_rows)
    drv.table.push(packer, drv.step())
    alloc = [rng.integers(8, 65, n_nodes) * 1000, rng.integers(32, 513, n_nodes) * GIB, rng.integers(0, 9, n_nodes)]
    over = [rng.integers(0, 3, n_nodes) * 250, rng.integers(0, 3, n_nodes) * (1 << 28), np.zeros(n_nodes, np.int64)]
    ig = rng.integers(0, 4, n_nodes).astype(np.int32)
    zid, rank = rng.integers(0, 3, n_nodes).astype(np.int32), rng.permutation(n_nodes).astype(np.int32)
    keys = list(drv.table.rrs)
    for s in range(2):
        for k in rng.choice(len(keys), len(keys) // 100, replace=False):     # 1 % of the rows rewritten
            cur = {n: (names[rng.integers(n_nodes)],) + r[1:] for n, r in drv.table.rrs[keys[k]].items()}
            drv.table.rr_set(keys[k], cur)
        drv.table.rr_set(("ns", f"new-{s}"), {f"e{j}": (names[j], 500, 1 << 28, 0) for j in range(21)})
        d = drv.step()
        assert d["reset"] is None
        drv.table.push(packer, d)
        ids = drv.table.node_ids(names)
        rnode, res = rv.to_usage_rows(drv.mirror, ids)
        want = packer.prepare_cluster_groups(alloc, over, rnode, res, ig, 4, zone_id=zid, n_zones=3, name_rank=rank)
        want_snap = packer.get_snapshot()
        got = packer.prepare_cluster_groups_resident(ids, alloc, over, ig, 4, zone_id=zid, n_zones=3, name_rank=rank)
        same((got, packer.get_snapshot()), (want, want_snap), (n_nodes, s))


def snapshot_state(p, apps):
    """what a held snapshot shows: its availability and an independent pack from it"""
    return p.get_snapshot(), p.pack_batch(apps, 0, native.MODE_INDEPENDENT)


def status_of(fn):
    return outcome(fn)[0]


def test_update_refusals_leave_the_table(gangpack):
    p = gangpack.GangPacker()
    try:
        d = dict(slot=[0], node_id=[0], cpu_milli=[1], mem_bytes=[1])
        assert status_of(lambda: p.reservation_table_update(d)) == INVALID                 # before any reset
        p.reservation_table_reset(8, 4)
        mirror = rv.ReservationMirror()
        first = dict(reset=dict(n_slots=8, n_node_ids=4), slot=np.arange(5, dtype=np.int32), node_id=np.array([0, 1, 2, 3, 1], np.int32),
                     cpu_milli=np.array([100, -7, 300, (1 << 61) - 1, 5], np.int64), mem_bytes=np.array([GIB, 2, 3, 4, -(1 << 50)], np.int64),
                     gpu=np.array([1, 0, 0, 2, 0], np.int64))
        p.reservation_table_update(first)
        mirror.apply(first)
        nodes = 4
        alloc = [np.full(nodes, 1 << 40), np.full(nodes, 1 << 40), np.full(nodes, 8)]

        def observe():
            ids = np.arange(nodes, dtype=np.int32)[::-1].copy()
            r = outcome(lambda: p.build_availability(alloc, None, *rv.to_usage_rows(mirror, ids)))
            got = outcome(lambda: (p.prepare_cluster_groups_resident(ids, alloc, None, None, 1), p.get_snapshot()))
            want = outcome(lambda: (p.prepare_cluster_groups(alloc, None, *rv.to_usage_rows(mirror, ids), None, 1), p.get_snapshot()))
            same(got, want, "observe")
            return r, got

        before = observe()
        bad = [
            (INVALID, dict(slot=[8], node_id=[0], cpu_milli=[1], mem_bytes=[1])),
            (INVALID, dict(slot=[-1], node_id=[0], cpu_milli=[1], mem_bytes=[1])),
            (INVALID, dict(slot=[5], node_id=[4], cpu_milli=[1], mem_bytes=[1])),
            (INVALID, dict(slot=[5], node_id=[-2], cpu_milli=[1], mem_bytes=[1])),
            (INVALID, dict(slot=[5, 6, 5], node_id=[0, 0, -1], cpu_milli=[1, 1, 1], mem_bytes=[1, 1, 1])),
            (INVALID, dict(slot=list(range(8)) + [0], node_id=[0] * 9, cpu_milli=[1] * 9, mem_bytes=[1] * 9)),
            (UNREPRESENTABLE, dict(slot=[0, 6], node_id=[0, 1], cpu_milli=[1, 1 << 61], mem_bytes=[1, 1])),
            (UNREPRESENTABLE, dict(slot=[6], node_id=[1], cpu_milli=[1], mem_bytes=[-(1 << 61)])),
            (UNREPRESENTABLE, dict(slot=[6], node_id=[1], cpu_milli=[1], mem_bytes=[1], gpu=[1 << 62])),
            (INVALID, dict(slot=[6], node_id=[1], cpu_milli=None, mem_bytes=[1])),
        ]
        for want, delta in bad:
            assert status_of(lambda: p.reservation_table_update(delta)) == want, delta
            same(observe(), before, delta)
        free = dict(slot=[2, 7], node_id=[-1, -1], cpu_milli=[1 << 62, 0], mem_bytes=[0, 0])      # a freed slot's values are not read
        p.reservation_table_update(free)
        mirror.apply(free)
        observe()
        assert status_of(lambda: p.reservation_table_reset(-1, 4)) == INVALID
        assert status_of(lambda: p.reservation_table_reset(1 << 31, 4)) == INVALID
        observe()                                                                           # a refused reset keeps the table
    finally:
        p.close()


def test_resident_entry_refusals_keep_the_snapshot(gangpack):
    p = gangpack.GangPacker()
    try:
        rng = np.random.default_rng(31)
        case = Case(2300, n=64, G=2, Z=3)
        c = case.c
        sa = sort_args(c)
        ids = np.arange(64, dtype=np.int32)
        assert status_of(lambda: p.prepare_cluster_groups_resident(ids, c["alloc"], c["over"], c["ig"], 2, *sa)) == INVALID  # no table
        p.prepare_cluster_groups(c["alloc"], c["over"], c["rnode"], c["res"], c["ig"], 2, *sa)
        apps = random_apps(rng, 30)
        held = snapshot_state(p, apps)
        p.reservation_table_reset(16, 64)
        p.reservation_table_update(dict(slot=[0, 1, 2], node_id=[3, 3, 9], cpu_milli=[1 << 60, 1 << 60, 5], mem_bytes=[0, 0, 1]))
        dup = ids.copy()
        dup[5] = 4
        out_of_range = ids.copy()
        out_of_range[7] = 64
        no_oh = ids.copy()
        cases = [
            (INVALID, dict(node_id=ids, overhead_node_id=no_oh)),                  # no overhead table
            (INVALID, dict(node_id=dup)),
            (INVALID, dict(node_id=out_of_range)),
            (INVALID, dict(node_id=np.full(64, -3, np.int32))),
            (UNREPRESENTABLE, dict(node_id=ids)),                                 # node 3: 2^61 reserved
        ]
        for want, kw in cases:
            for entry in ("groups", "zones", "resched"):
                st = status_of(lambda: resident_call(p, case, entry, **kw))
                assert st == want, (entry, want)
            same(snapshot_state(p, apps), held, want)
        # overhead ids: out of range, given twice, and a per-node overhead sum >= 2^61
        p.overhead_table_reset(n_slots=4, n_node_ids=8, n_app_keys=1, n_app_ids=1, n_names=1)
        p.overhead_table_update(dict(slot=[0, 1], node_id=[2, 2], req_cpu_milli=[1 << 60, 1 << 60], req_mem_bytes=[0, 0],
                                     listed=[1, 1], app_key=[-1, -1], app_id=[-1, -1], name_id=[0, 0]))
        safe = np.where(ids == 3, -1, ids).astype(np.int32)
        oid = np.full(64, -1, np.int32)
        for want, o in [(INVALID, [8]), (INVALID, [1, 1]), (UNREPRESENTABLE, [2])]:
            oo = oid.copy()
            oo[10:10 + len(o)] = o
            for entry in ("groups", "zones", "resched"):
                assert status_of(lambda: resident_call(p, case, entry, node_id=safe, overhead_node_id=oo)) == want, (entry, o)
            same(snapshot_state(p, apps), held, o)
    finally:
        p.close()


def resident_call(p, case, entry, node_id, overhead_node_id=None):
    c = case.c
    sa = sort_args(c)
    over = None if overhead_node_id is not None else c["over"]
    if entry == "groups":
        return p.prepare_cluster_groups_resident(node_id, c["alloc"], over, c["ig"], 2, *sa, overhead_node_id=overhead_node_id)
    if entry == "zones":
        return p.prepare_cluster_zones_groups_resident(node_id, c["alloc"], over, c["ig"], 2, *sa, overhead_node_id=overhead_node_id)
    exe = (np.array([500]), np.array([GIB]))
    return p.reschedule_from_reservations_resident(node_id, c["alloc"], over, exe, zone_id=sa[0], n_zones=sa[1], name_rank=sa[2],
                                                   overhead_node_id=overhead_node_id)


@pytest.mark.parametrize("top", [(1 << 60) - 1, 1 << 60])
def test_domain_edges(packer, top):
    """two rows on one node summing to 2^61 - 1 (exact) or 2^61 (refused), negative rows at the mirror image"""
    for sign in (1, -1):
        packer.reservation_table_reset(4, 2)
        d = dict(reset=dict(n_slots=4, n_node_ids=2), slot=np.array([0, 1, 2], np.int32), node_id=np.array([1, 1, 0], np.int32),
                 cpu_milli=np.array([sign * (1 << 60), sign * top, 1], np.int64), mem_bytes=np.array([0, 0, 2], np.int64))
        packer.reservation_table_update(d)
        mirror = rv.ReservationMirror()
        mirror.apply(d)
        ids = np.array([1, 0], np.int32)
        alloc = [np.zeros(2, np.int64), np.full(2, GIB)]
        rnode, res = rv.to_usage_rows(mirror, ids)
        a = outcome(lambda: (packer.prepare_cluster_groups(alloc, None, rnode, res, None, 1), packer.get_snapshot()))
        b = outcome(lambda: (packer.prepare_cluster_groups_resident(ids, alloc, None, None, 1), packer.get_snapshot()))
        same(a, b, (top, sign))
        assert a[0] == (0 if top < 1 << 60 else UNREPRESENTABLE), (top, sign)


def test_independence(gangpack):
    """table updates leave a held snapshot and gp_last_stats alone; a live table changes no per-call entry's results;
    gp_destroy with both tables live"""
    p, alone = gangpack.GangPacker(), gangpack.GangPacker()
    try:
        rng = np.random.default_rng(41)
        case = Case(2400, n=200, G=2, Z=3)
        c = case.c
        sa = sort_args(c)
        apps = random_apps(rng, 40)
        run = lambda q: (q.prepare_cluster_groups(c["alloc"], c["over"], c["rnode"], c["res"], c["ig"], 2, *sa), snapshot_state(q, apps),
                         q.stats(), q.reschedule_from_reservations(c["alloc"], c["over"], c["rnode"], c["res"], (np.array([500]), np.array([GIB]))))
        base = run(alone)
        p.prepare_cluster_groups(c["alloc"], c["over"], c["rnode"], c["res"], c["ig"], 2, *sa)
        held = snapshot_state(p, apps)
        stats = p.stats()
        drv = Driver()
        for d in stream(case, drv, rng, steps=4, per_step=5):
            drv.table.push(p, d)
            assert p.stats() == stats
        same(snapshot_state(p, apps), held, "held")
        p.overhead_table_reset(n_slots=4, n_node_ids=4, n_app_keys=1, n_app_ids=1, n_names=1)
        got = run(p)
        same((got[0], got[1], got[3]), (base[0], base[1], base[3]), "per-call with live tables")
    finally:
        p.close()                                                        # both tables live
        alone.close()
