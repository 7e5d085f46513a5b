"""The resident overhead table on the device (gp_overhead_table_reset / _update / _query).

After every update the query must equal, bit for bit, gp_node_overhead on the equivalent encoding of the table
(overhead.to_encoding of the numpy mirror), the numpy evaluator and the string restatement: over random event streams, full
synthetic clusters up to 50 000 nodes x 1 000 000 records with 1 % churn, and enough insert/remove cycles to rehash the
member set several times.  Then every refusal of an update (the table unchanged after it), sums just below and at 2^61,
calls before any reset, and a table that leaves every other entry of the context untouched."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import overhead as oh
from test_overhead_model import pod
from test_overhead_table_model import Driver, churn, lists

pytestmark = pytest.mark.gpu

SPARK = "spark-scheduler"


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def same(a, b):
    """two (overhead, nonsched, has_reservation, n_warned) answers, bit for bit"""
    assert lists(a[0]) == lists(b[0]) and lists(a[1]) == lists(b[1])
    assert np.array_equal(a[2], b[2]) and a[3] == b[3]


def device_check(packer, drv, nodes, restated=True):
    """the device query == gp_node_overhead on the mirror's encoding == the evaluator (== the restatement)"""
    ids = drv.table.node_ids(nodes)
    ids = ids[ids >= 0]
    got = packer.overhead_table_query(ids)
    enc = oh.to_encoding(drv.mirror, ids)
    same(got, packer.node_overhead(enc))
    same(got, oh.evaluate(enc))
    if restated:
        drv.check(nodes, query=packer.overhead_table_query)
    return got


def step(packer, drv):
    d = drv.step()
    drv.table.push(packer, d)
    return d


@pytest.mark.parametrize("seed", range(10))
def test_random_churn_streams(packer, seed):
    rng = np.random.default_rng(900 + seed)
    n_nodes = 1 + seed % 6
    drv = Driver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
    nodes = [f"n{i}" for i in range(n_nodes)]
    for d in churn(rng, drv, n_nodes, steps=30, per_step=1 + seed % 7):
        drv.table.push(packer, d)
        device_check(packer, drv, nodes)
    assert drv.replays >= 2


def load_cluster(drv, nodes, pods, lister, rrs, soft):
    for p in pods:
        drv.pod_event("add", p)
    for p in lister.values():
        drv.table.lister_set(p)
    for k, v in rrs.items():
        drv.table.rr_set(k, v)
    for k, v in soft.items():
        drv.table.soft_set(k, v)


@pytest.mark.parametrize("n_nodes,n_pods,big,huge", [(10_000, 300_000, 20, 0), (50_000, 1_000_000, 40, 100_000)])
def test_synthetic_clusters_with_churn(packer, n_nodes, n_pods, big, huge):
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(n_nodes, n_nodes, n_pods, big_apps=big, huge_app=huge)
    drv = Driver(n_slots=n_pods, n_node_ids=n_nodes, n_app_keys=1 << 16, n_app_ids=1 << 16, n_names=1 << 21)
    load_cluster(drv, nodes, pods, lister, rrs, soft)
    step(packer, drv)
    t = drv.table

    def against_views():
        got = t.answer(nodes, packer.overhead_table_query)
        want = packer.node_overhead(oh.encode(t.slots, t.lister, t.rrs, t.soft, nodes))
        same(got[:2] + (got[2][:len(t.slots)], got[3]), want)
        device_check(packer, drv, nodes, restated=False)
        return got

    first = against_views()
    assert first[3] > 0 and 0 < first[2].sum() < n_pods
    rng = np.random.default_rng(3)
    for s in range(3):                                            # 1 % of the records rewritten, one new RR of 20 pods
        for i in rng.choice(len(pods), len(pods) // 100, replace=False):
            p = pods[i]
            drv.pod_event("delete", p)
            q = dict(p, uid=f"{p['uid']}-{s}", nodeName=nodes[rng.integers(len(nodes))])
            drv.pod_event("add", q)
            pods[i] = q
            if rng.random() < 0.1:
                t.lister_delete(q["namespace"], q["name"])
        t.rr_set((f"ns-{s}", f"churn-{s}"), [f"churn-{s}-exec-{e}" for e in range(20)])
        d = step(packer, drv)
        assert d["reset"] is None
        against_views()


def test_member_set_rehashes(packer):
    """Cycles that replace ~350 of ~400 members: following the documented rule (1024 cells after a reset; an update whose
    insertions could take keys + tombstones past half the cells first rehashes into max(cells, pow2 >= 4 * (keys +
    insertions))) over the deltas' exact counts, the set is rebuilt several times; the answers stay those of the mirror."""
    drv = Driver()
    nodes = ["n1", "n2"]
    for k in range(50):
        p = pod("a", f"x-{k}", nodes[k % 2], 10 + k, 1, labels={"spark-app-id": "big", "spark-role": "executor"}, sched=SPARK)
        drv.pod_event("add", p)
        drv.table.lister_set(p)
    drv.table.rr_set(("a", "big"), [])
    step(packer, drv)
    cells, keys, used, rehashes = 1024, 0, 0, 0
    for cycle in range(24):
        names = [f"x-{k}" for k in range(50)] + [f"c{cycle}-{j}" for j in range(350)]
        for kind_set in (drv.table.rr_set, drv.table.soft_set):
            key = ("a", "big") if kind_set is drv.table.rr_set else "big"
            kind_set(key, names[:200] if kind_set is drv.table.rr_set else names[200:])
        d = step(packer, drv)
        ins = int(d["member_present"].sum())
        rem = len(d["member_present"]) - ins
        if 2 * (used + ins) > cells:
            rehashes += 1
            need = 1024
            while need < 4 * (keys + ins):
                need *= 2
            cells, used = max(cells, need), keys
        keys += ins - rem
        used += ins
        device_check(packer, drv, nodes)
    assert rehashes >= 3


def test_update_refusals_leave_the_table_unchanged(packer, gangpack):
    drv = Driver()
    nodes = ["n1", "n2"]
    rng = np.random.default_rng(5)
    for d in churn(rng, drv, 2, steps=4, per_step=20):
        drv.table.push(packer, d)
    size = drv.table.size
    before = device_check(packer, drv, nodes)
    ids = drv.table.node_ids(nodes)
    ids = ids[ids >= 0]

    def base():
        return dict(reset=None, slot=np.array([0, 1], np.int32), node_id=np.array([0, 0], np.int32),
                    req_cpu_milli=np.array([5, 6], np.int64), req_mem_bytes=np.array([1, 1], np.int64),
                    req_gpu=np.array([0, 0], np.int64), listed=np.array([1, 1], np.uint8), app_key=np.array([0, -1], np.int32),
                    app_id=np.array([0, -1], np.int32), name_id=np.array([0, 1], np.int32), is_executor=np.array([1, 0], np.uint8),
                    spark_scheduler=np.array([1, 0], np.uint8), rr_app_key=np.array([0, 1], np.int32),
                    rr_exists=np.array([1, 0], np.uint8), member_kind=np.array([0, 1], np.uint8),
                    member_app=np.array([0, 0], np.int32), member_name=np.array([0, 0], np.int32),
                    member_present=np.array([1, 1], np.uint8))

    def put(k, i, v):
        return lambda d: d[k].__setitem__(i, v)

    cases = [
        ("slot out of range", put("slot", 1, size["n_slots"]), 1, "out of its range"),
        ("negative slot", put("slot", 0, -1), 1, "out of its range"),
        ("slot twice", put("slot", 1, 0), 1, "given twice"),
        ("node id out of range", put("node_id", 0, size["n_node_ids"]), 1, "out of its range"),
        ("node id below -1", put("node_id", 0, -2), 1, "out of its range"),
        ("app key out of range", put("app_key", 0, size["n_app_keys"]), 1, "out of its range"),
        ("app id out of range", put("app_id", 0, size["n_app_ids"]), 1, "out of its range"),
        ("name out of range", put("name_id", 1, size["n_names"]), 1, "out of its range"),
        ("app key without app id", put("app_id", 0, -1), 1, "disagree"),
        ("negative request", put("req_mem_bytes", 1, -1), 1, "negative request"),
        ("negative gpu request", put("req_gpu", 0, -3), 1, "negative request"),
        ("request at 2^61", put("req_cpu_milli", 0, 1 << 61), 6, "request >= 2\\^61"),
        ("rr app key twice", put("rr_app_key", 1, 0), 1, "given twice"),
        ("rr app key out of range", put("rr_app_key", 0, size["n_app_keys"]), 1, "out of its range"),
        ("member kind 2", put("member_kind", 0, 2), 1, "out of its range"),
        ("kind-1 app past the app ids", put("member_app", 1, size["n_app_ids"]), 1, "out of its range"),
        ("member name out of range", put("member_name", 0, -1), 1, "out of its range"),
        ("member triple twice", lambda d: (put("member_kind", 1, 0)(d)), 1, "given twice"),
        ("missing column", lambda d: d.__setitem__("app_key", None), 1, "missing arrays"),
        ("negative count", lambda d: d.__setitem__("n_member", -1), 1, "negative counts"),
    ]
    for name, mutate, status, msg in cases:
        d = base()
        mutate(d)
        with pytest.raises(gangpack.GangpackError, match=msg) as ei:
            packer.overhead_table_update(d)
        assert ei.value.status == status, name
        same(packer.overhead_table_query(ids), before)


def test_sums_just_below_and_at_2_61(packer, gangpack):
    top = (1 << 61) - 1
    packer.overhead_table_reset(n_slots=3, n_node_ids=1, n_app_keys=1, n_app_ids=1, n_names=3)

    def write(slots, cpu):
        n = len(slots)
        packer.overhead_table_update(dict(slot=np.array(slots, np.int32), node_id=np.zeros(n, np.int32),
                                          req_cpu_milli=np.array(cpu, np.int64), req_mem_bytes=np.zeros(n, np.int64),
                                          app_key=np.full(n, -1, np.int32), app_id=np.full(n, -1, np.int32),
                                          name_id=np.arange(n, dtype=np.int32)))

    write([0, 1], [1 << 60, (1 << 60) - 1])
    ov, ns, _, _ = packer.overhead_table_query([0])
    assert int(ov[0][0]) == int(ns[0][0]) == top
    write([2], [1])                                               # the sum reaches 2^61 at query time
    with pytest.raises(gangpack.GangpackError, match="sum >= 2\\^61") as ei:
        packer.overhead_table_query([0])
    assert ei.value.status == 6
    packer.overhead_table_update(dict(slot=np.array([1], np.int32), node_id=np.array([-1], np.int32),
                                      req_cpu_milli=np.zeros(1, np.int64), req_mem_bytes=np.zeros(1, np.int64),
                                      app_key=np.full(1, -1, np.int32), app_id=np.full(1, -1, np.int32),
                                      name_id=np.zeros(1, np.int32)))   # freeing a slot brings the query back
    ov, _, has, warned = packer.overhead_table_query([0])
    assert int(ov[0][0]) == (1 << 60) + 1 and has.tolist() == [0, 0, 0] and warned == 0
    with pytest.raises(gangpack.GangpackError, match="node id out of range"):
        packer.overhead_table_query([1])
    with pytest.raises(gangpack.GangpackError, match="given twice"):
        packer.overhead_table_query([0, 0])


def test_calls_before_any_reset(gangpack):
    p = gangpack.GangPacker()
    try:
        with pytest.raises(gangpack.GangpackError, match="no overhead table") as ei:
            p.overhead_table_query([0])
        assert ei.value.status == 1
        with pytest.raises(gangpack.GangpackError, match="no overhead table") as ei:
            p.overhead_table_update(dict(slot=np.zeros(0, np.int32)))
        assert ei.value.status == 1
        p.overhead_table_reset(n_slots=0, n_node_ids=0, n_app_keys=0, n_app_ids=0, n_names=0)
        ov, _, has, warned = p.overhead_table_query([])
        assert len(ov[0]) == 0 and len(has) == 0 and warned == 0
        with pytest.raises(gangpack.GangpackError, match="negative capacity"):
            p.overhead_table_reset(n_slots=-1, n_node_ids=0, n_app_keys=0, n_app_ids=0, n_names=0)
        p.overhead_table_query([])                                # a refused reset keeps the table
    finally:
        p.close()


def test_refused_reset_keeps_a_nonempty_table(gangpack):
    """A reset refused over a table of 1000 slots keeps that table: a query still answers as before, has_reservation over
    the same 1000 slots"""
    p = gangpack.GangPacker()
    try:
        drv = Driver(n_slots=1000, n_node_ids=8, n_app_keys=8, n_app_ids=8, n_names=1024)
        for k in range(600):
            q = pod("a", f"e-{k}", f"n{k % 5}", 10 + k, 1, labels={"spark-app-id": "app", "spark-role": "executor"},
                    sched=SPARK, uid=f"u{k}")
            drv.pod_event("add", q)
            drv.table.lister_set(q)
        drv.table.rr_set(("a", "app"), [f"e-{k}" for k in range(0, 600, 3)])
        drv.table.push(p, drv.step())
        ids = np.arange(5, dtype=np.int32)
        before = p.overhead_table_query(ids)
        assert len(before[2]) == 1000 and before[2].sum() == 200
        for size in (dict(n_slots=4, n_node_ids=1, n_app_keys=1, n_app_ids=1, n_names=-1),
                     dict(n_slots=1 << 31, n_node_ids=1, n_app_keys=1, n_app_ids=1, n_names=1)):
            with pytest.raises(gangpack.GangpackError) as ei:
                p.overhead_table_reset(**size)
            assert ei.value.status == 1
            same(p.overhead_table_query(ids), before)
        same(before, p.node_overhead(oh.to_encoding(drv.mirror, ids)))
    finally:
        p.close()


def test_table_leaves_the_other_entries_alone(gangpack):
    """The same calls on a context with a live table and on one without: equal outputs; the table's answers unchanged"""
    from k8s_spark_scheduler_b200 import synth
    g = gangpack
    nodes = synth.make_nodes(256, groups=1)
    apps = synth.make_apps(64, groups=1, young_frac=0.0)
    eoff, eorder = synth.group_orders(nodes)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group", "young")}
    names, rec, lister, rrs, soft, pods = oh.synthetic_cluster(11, 256, 20_000, big_apps=2)
    enc = oh.encode(rec.slots, lister, rrs, soft, names)
    rng = np.random.default_rng(4)
    n = 256
    alloc = (rng.integers(64, 129, n).astype(np.int64) * 1000, rng.integers(256, 513, n).astype(np.int64) << 30,
             rng.integers(0, 9, n).astype(np.int64))
    res_node = rng.integers(0, n, 300).astype(np.int32)
    res = (rng.integers(0, 4000, 300).astype(np.int64), rng.integers(0, 8, 300).astype(np.int64) << 30, np.zeros(300, np.int64))

    def run(p):
        out = []
        p.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
        out.append(p.pack_batch(a, g.TIGHTLY_PACK, g.MODE_INDEPENDENT))
        out.append(p.get_snapshot())
        out.append(p.node_overhead(enc))
        out.append((p.prepare_cluster(alloc, None, res_node, res),))
        out.append(p.pack_batch(a, g.DISTRIBUTE_EVENLY, g.MODE_INDEPENDENT))
        out.append(p.get_snapshot())
        return out

    def flat(xs):
        for x in xs:
            if isinstance(x, (tuple, list)):
                yield from flat(x)
            else:
                yield np.asarray(x)

    plain = gangpack.GangPacker()
    with_table = gangpack.GangPacker()
    try:
        drv = Driver()
        load_cluster(drv, names, pods, lister, rrs, soft)
        drv.table.push(with_table, drv.step())
        ids = drv.table.node_ids(names)
        ids = ids[ids >= 0]
        before = with_table.overhead_table_query(ids)
        want, got = run(plain), run(with_table)
        assert all(np.array_equal(x, y) for x, y in zip(flat(want), flat(got)))
        same(with_table.overhead_table_query(ids), before)
        same(before, plain.node_overhead(oh.to_encoding(drv.mirror, ids)))
    finally:
        plain.close()
        with_table.close()                                        # gp_destroy with a live table

