"""The node-table forms of the failover reconciler and the unschedulable-pod marker (gp_reconcile_find_nodes_node_table,
gp_exceeds_cluster_capacity_node_table, gp_exceeds_cluster_capacity_affinity_node_table) and the node table's creation column.

After every flush of seeded node, label, reservation and overhead churn, each node-table entry must give what its resident
entry gives on the columns decoded from the numpy mirrors (nodes.NodeMirror.to_columns, nodes.label_columns,
nodes.reconcile_groups) -- bit for bit: placed, executor nodes, availability, exceeds, affinity errors and the status.  One
small reconcile is also checked against the literal restatement of tests/reconcile_ref.py.  Every refusal of the gather is
hit once, and the tables and the held snapshot are checked unchanged afterwards.  The three Predicate node-table entries
give the same results whether or not creation times were written."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import native, nodes
from test_gpu_node_table import GROUPS, ZONES, World, outcome, same
import reconcile_ref

pytestmark = pytest.mark.gpu

INVALID = 1
IG = "instance-group"
RECON_GROUPS = GROUPS + ["gx", "gz"]             # "gz": a group no node carries
PACKERS = range(5)
AFFS = [{"required": [{"matchExpressions": [(IG, "In", ["g0", "g1"])]}]},
        {"required": [{"matchExpressions": [(nodes.ZONE_LABEL, "NotIn", ["z1"])]}]},
        {"required": [{"matchExpressions": [(IG, "DoesNotExist", [])]}]}]


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


class CWorld(World):
    """World with creation times (few distinct values: equal times are common), nodes labelled "" for the instance group,
    and more unschedulable and not-ready nodes"""

    def node_event(self, name):
        r = self.rng
        lab = {}
        if r.random() < 0.85:
            lab[nodes.ZONE_LABEL] = ZONES[r.integers(len(ZONES))]
        u = r.random()
        if u < 0.7:
            lab[IG] = (GROUPS + ["gx"])[r.integers(len(GROUPS) + 1)]
        elif u < 0.8:
            lab[IG] = ""
        self.labels.set_node(name, lab)
        alloc = (int(r.integers(2, 5)) * 16000, int(r.integers(2, 5)) * (64 << 30), int(r.integers(0, 3)))
        self.table.set_node(name, alloc, r.random() < 0.08, r.random() < 0.92, creation=int(r.integers(0, 6)) * 10 ** 9)


def defined(r):
    """a reconcile result with the executor-node entries past placed[i] (undefined) set to -1"""
    placed, execn, off, avail = r
    keep = np.full(len(execn), -1, np.int32)
    for i, k in enumerate(placed):
        keep[off[i]:off[i] + max(int(k), 0)] = execn[off[i]:off[i] + max(int(k), 0)]
    return placed, keep, off, avail


def recon_args(w):
    return nodes.reconcile_label_args(w.labels, IG, RECON_GROUPS)


def recon_apps(rng, q, G):
    return dict(exe_cpu=rng.integers(1, 9, q) * 2000, exe_mem=rng.integers(1, 17, q) * (1 << 30),
                exe_gpu=(rng.integers(0, 4, q) == 0).astype(np.int64), count=rng.integers(0, 5, q).astype(np.int32),
                group=rng.integers(0, G, q).astype(np.int32))


def marker_apps(rng, q, lo, hi):
    return dict(drv_cpu=rng.integers(1, 5, q) * 1000, drv_mem=rng.integers(1, 9, q) * (1 << 30), drv_gpu=np.zeros(q, np.int64),
                exe_cpu=rng.integers(1, 17, q) * 1000, exe_mem=rng.integers(1, 33, q) * (1 << 30),
                exe_gpu=(rng.integers(0, 5, q) == 0).astype(np.int64), count=rng.integers(0, 60, q).astype(np.int32),
                group=rng.integers(lo, hi, q).astype(np.int32))


def check_reconcile(p, w, label, names=None, zone=True, q=40):
    names = w.listed() if names is None else names
    nd = w.nodes_dict(names, priorities=False, zone=zone)
    ra = recon_args(w)
    ndr = dict(nd, instance_group_key=ra["instance_group_key"], instance_group_value=ra["instance_group_value"])
    cols, _ = w.decoded(nd)
    grp = nodes.reconcile_groups(w.labels.mirror, nd["node_table_id"], **ra)
    G, miss = ra["n_groups"], ra["instance_group_missing"]
    apps = recon_apps(w.rng, q, G)
    a = outcome(lambda: defined(p.reconcile_find_nodes_resident(nd["reservation_id"], cols["alloc"], None, grp, cols["creation"], apps,
                                                                G, unschedulable=cols["unschedulable"], ready=cols["ready"],
                                                                overhead_node_id=nd["overhead_node_id"])))
    igo = np.full(len(names), -9, np.int32)
    b = outcome(lambda: defined(p.reconcile_find_nodes_node_table(dict(ndr, instance_group_out=igo), apps, G, miss)))
    same(a, b, (label, "reconcile"))
    assert a[0] == 0, (label, a[0])
    if len(names):
        assert np.array_equal(igo, grp)
    return a


def check_marker(p, w, label, names=None, zone=True, packers=PACKERS, q=30):
    names = w.listed() if names is None else names
    nd = w.nodes_dict(names, priorities=False, zone=zone)
    cols, lab = w.decoded(nd)
    zk = dict(zone_id=lab["zone_id"], n_zones=nd["n_zones"] if lab["zone_id"] is not None else 1)
    rng = w.rng
    node_group = rng.integers(-1, 2, len(names)).astype(np.int32)
    enc = w.labels.encode_affinities(AFFS, names)
    oid = nd["overhead_node_id"]
    for pk in packers:
        apps = marker_apps(rng, q, -1, 2)
        a = outcome(lambda: p.exceeds_cluster_capacity_resident(cols["alloc"], oid, apps, pk, node_group=node_group, n_groups=2, **zk))
        no_res = {k: v for k, v in nd.items() if k != "reservation_id"} if pk % 2 else nd
        b = outcome(lambda: p.exceeds_cluster_capacity_node_table(no_res, apps, pk, node_group, 2))
        same(a, b, (label, "marker", pk))
        assert a[0] == 0, (label, pk, a[0])
        aapps = marker_apps(rng, q, 0, len(AFFS))
        a = outcome(lambda: p.exceeds_cluster_capacity_affinity_label_table(cols["alloc"], oid, nd["node_table_id"], enc, aapps, pk, **zk))
        b = outcome(lambda: p.exceeds_cluster_capacity_affinity_node_table(nd, enc, aapps, pk))
        same(a, b, (label, "affinity marker", pk))
        assert a[0] == 0, (label, pk, a[0])


@pytest.mark.parametrize("seed,n", [(1, 200), (2, 120)])
def test_churn_identity(packer, seed, n):
    w = CWorld(seed, n)
    placed = 0
    for s in range(8):
        w.churn(n // 3 if s == 0 else max(4, n // 20))
        w.flush(packer)
        zone = s % 3 != 1
        got = check_reconcile(packer, w, (seed, s), zone=zone)
        placed += int((got[1][0] > 0).sum())
        check_marker(packer, w, (seed, s), zone=zone)
    assert placed > 0
    c = w.table.mirror.to_columns(w.table.node_ids(list(w.table.nodes)))
    assert len(np.unique(c["creation"])) < len(c["creation"])          # equal creation times were met
    assert c["unschedulable"].any() and not c["ready"].all()


def test_empty_node_list_and_no_drivers(packer):
    w = CWorld(5, 40)
    w.churn(40)
    w.flush(packer)
    check_reconcile(packer, w, "no nodes", names=[])
    check_reconcile(packer, w, "no drivers", q=0)
    check_marker(packer, w, "no nodes", names=[], packers=(0, 3))
    check_marker(packer, w, "no drivers", q=0, packers=(1, 4))


def test_churn_identity_50000_nodes(packer):
    w = CWorld(11, 50000)
    w.churn(50000)
    w.flush(packer)
    check_reconcile(packer, w, "50k", q=200)
    check_marker(packer, w, "50k", packers=(2, 4), q=1000)
    w.churn(500)                                      # 1 % churn
    w.flush(packer)
    check_reconcile(packer, w, "50k after churn", names=w.listed(False), q=200)


def test_small_reconcile_against_the_literal(gangpack):
    from k8s_spark_scheduler_b200 import affinity
    rng = np.random.default_rng(3)
    p = gangpack.GangPacker()
    try:
        labels = affinity.LabelTable(n_node_ids=8)
        table = nodes.NodeTable(labels, n_node_ids=8)
        n = 14
        names = [f"m{i:02d}" for i in range(n)]
        vals = [None if i % 5 == 0 else ["a", "b", ""][i % 3] for i in range(n)]
        alloc = (rng.integers(2, 5, n) * 8000, rng.integers(2, 5, n) * (16 << 30), rng.integers(0, 2, n))
        uns, rdy = (rng.random(n) < 0.15).astype(np.uint8), (rng.random(n) < 0.85).astype(np.uint8)
        creation = rng.integers(0, 3, n) * 7
        for i, nm in enumerate(names):
            labels.set_node(nm, {} if vals[i] is None else {IG: vals[i]})
            table.set_node(nm, tuple(int(a[i]) for a in alloc), bool(uns[i]), bool(rdy[i]), creation=int(creation[i]))
        labels.flush(p)
        table.flush(p)
        r = 6
        res_node = rng.integers(0, n, r).astype(np.int32)
        res = (rng.integers(0, 4, r) * 1000, rng.integers(0, 4, r) * (1 << 30), np.zeros(r, np.int64))
        p.reservation_table_reset(n_slots=r, n_node_ids=n)
        p.reservation_table_update(dict(slot=np.arange(r, dtype=np.int32), node_id=res_node, cpu_milli=res[0], mem_bytes=res[1], gpu=res[2]))
        p.overhead_table_reset(n_slots=1, n_node_ids=1, n_app_keys=1, n_app_ids=1, n_names=1)
        order = list(rng.permutation(n))                 # the lister's order
        listed = [names[i] for i in order]
        ra = nodes.reconcile_label_args(labels, IG, ["b", "a", "zz"])
        groups = ["b", "a", "zz", ""]
        q = 10
        dgroup = [groups[int(rng.integers(0, 4))] for _ in range(q)]
        exe = (rng.integers(1, 6, q) * 1000, rng.integers(1, 9, q) * (1 << 30), np.zeros(q, np.int64))
        mn, running = rng.integers(0, 6, q), rng.integers(0, 3, q)
        case = dict(names=listed, alloc=tuple(a[order] for a in alloc), label=[vals[i] for i in order], unschedulable=uns[order],
                    ready=rdy[order], creation=creation[order], overhead=None,
                    res_node=np.array([order.index(int(x)) for x in res_node], np.int32), res=res,
                    dgroup=dgroup, exe=exe, min=mn, running=running)
        want_placed, want_names, want_final = reconcile_ref.literal(case)
        nd = dict(node_table_id=table.node_ids(listed), reservation_id=np.array(order, np.int32),
                  overhead_node_id=np.full(n, -1, np.int32), instance_group_key=ra["instance_group_key"],
                  instance_group_value=ra["instance_group_value"])
        count = np.maximum(0, mn - np.minimum(running, mn)).astype(np.int32)
        apps = dict(exe_cpu=exe[0], exe_mem=exe[1], exe_gpu=exe[2], count=count,
                    group=np.array([groups.index(g) for g in dgroup], np.int32))
        placed, execn, off, avail = p.reconcile_find_nodes_node_table(nd, apps, ra["n_groups"], ra["instance_group_missing"])
        assert list(placed) == want_placed
        for i in range(q):
            assert [listed[j] for j in execn[off[i]:off[i] + max(placed[i], 0)]] == want_names[i], i
        assert [tuple(int(avail[d][j]) for d in range(3)) for j in range(n)] == [tuple(want_final[nm]) for nm in listed]
        assert (np.asarray(placed) == -1).any() and (np.asarray(placed) > 0).any()
    finally:
        p.close()


def test_refusals_leave_tables_and_snapshot(gangpack):
    p = gangpack.GangPacker()
    try:
        w = CWorld(31, 60)
        w.churn(60)
        w.flush(p)
        names = w.listed(False)
        nd = w.nodes_dict(names, priorities=False)
        ra = recon_args(w)
        ndr = dict(nd, instance_group_key=ra["instance_group_key"], instance_group_value=ra["instance_group_value"])
        G, miss = ra["n_groups"], ra["instance_group_missing"]
        apps = recon_apps(np.random.default_rng(1), 20, G)
        mapps = marker_apps(np.random.default_rng(2), 20, -1, 1)
        enc = w.labels.encode_affinities(AFFS, names)
        aapps = marker_apps(np.random.default_rng(3), 20, 0, len(AFFS))
        p.prepare_cluster_groups_node_table(nd, None, len(GROUPS))         # the held snapshot
        snap = p.get_snapshot()

        def answers():
            return (defined(p.reconcile_find_nodes_node_table(ndr, apps, G, miss)), p.exceeds_cluster_capacity_node_table(nd, mapps, 2),
                    p.exceeds_cluster_capacity_affinity_node_table(nd, enc, aapps, 3))
        good = answers()
        grp = nodes.reconcile_groups(w.labels.mirror, nd["node_table_id"], **ra)
        assert (grp == miss).any()                                            # some node has no label, or ""
        lacking = [i for i, nm in enumerate(names) if IG not in w.labels.labels[nm]]
        assert lacking
        ids = nd["node_table_id"]
        dup, absent = ids.copy(), ids.copy()
        dup[1] = dup[0]
        absent[0] = w.table.size["n_node_ids"] - 1 if w.table.size["n_node_ids"] - 1 not in set(ids.tolist()) else -3
        carried = [g for g in np.unique(grp) if g != miss]
        unlisted = ra["instance_group_value"].copy()
        unlisted[carried[0]] = -99
        lab = nodes.label_columns(w.labels.mirror, **nd)
        zcar = [z for z in np.unique(lab["zone_id"]) if z != nd["zone_missing"]]
        zunl = nd["zone_value"].copy()
        zunl[zcar[0]] = -99
        node_cases = [("duplicate id", dict(node_table_id=dup)), ("absent id", dict(node_table_id=absent)),
                      ("unlisted zone", dict(zone_value=zunl))]
        recon_cases = node_cases + [("unlisted group", dict(instance_group_value=unlisted)),
                                    ("missing label, -1", dict(_missing=-1)), ("missing out of range", dict(_missing=G))]
        with pytest.raises(ValueError):                                          # a value list shorter than n_groups
            p.reconcile_find_nodes_node_table(dict(ndr, instance_group_value=ndr["instance_group_value"][:-1]), apps, G, miss)
        for what, ch in recon_cases:
            m = ch.pop("_missing", miss)
            assert outcome(lambda: p.reconcile_find_nodes_node_table(dict(ndr, **ch), apps, G, m))[0] == INVALID, what
            same(p.get_snapshot(), snap, what)
        for what, ch in node_cases:
            assert outcome(lambda: p.exceeds_cluster_capacity_node_table(dict(nd, **ch), mapps, 2))[0] == INVALID, what
            assert outcome(lambda: p.exceeds_cluster_capacity_affinity_node_table(dict(nd, **ch), enc, aapps, 3))[0] == INVALID, what
            same(p.get_snapshot(), snap, what)
        same(answers(), good, "after the refusals")
        # a node-table id past the table: reset it behind the mirror, then replay
        p.node_table_reset(n_node_ids=0)
        assert outcome(lambda: p.reconcile_find_nodes_node_table(ndr, apps, G, miss))[0] == INVALID
        w.table.replay()
        w.table.flush(p)
        same(answers(), good, "after replay")
        same(p.get_snapshot(), snap, "after replay")
    finally:
        p.close()


def test_predicate_entries_ignore_creation(gangpack):
    p = gangpack.GangPacker()
    try:
        w = CWorld(41, 150)
        w.churn(150)
        w.flush(p)
        names = w.listed()
        nd = w.nodes_dict(names)
        exe = (np.arange(1, 13) * 1500, np.arange(1, 13) * (1 << 30))

        def run():
            out = [p.prepare_cluster_groups_node_table(nd, None, len(GROUPS)), p.get_snapshot()]
            for kind in (native.LAYOUT_AZ_AWARE, native.LAYOUT_SINGLE_AZ):
                out += [p.prepare_cluster_zones_groups_node_table(nd, None, len(GROUPS), kind=kind), p.get_snapshot()]
            out += [p.reschedule_from_reservations_node_table(nd, exe, min_frag=mf) for mf in (False, True)]
            return out
        assert w.table.mirror.creation.any()
        with_creation = run()
        w.table.replay()
        d = w.table.delta()
        p.node_table_reset(**d["reset"])
        p.node_table_update({k: v for k, v in d.items() if k not in ("reset", "creation")})   # creation NULL: 0 everywhere
        same(run(), with_creation, "creation not written")
        w.table.replay()
        w.table.flush(p)
        same(run(), with_creation, "creation written again")
    finally:
        p.close()
