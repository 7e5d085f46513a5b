"""gp_node_overhead on the device.

The per-node sums, has_reservation and the warning count are checked bit for bit against the string restatement
(tests/overhead_ref.py) and the numpy evaluator of the encoded arrays, from hand-derived vectors up to 50 000 nodes x 1 000 000
pods with one application of 100 000 reserved pods; then free slots, sums just below and at 2^61, every refusal, an untouched
context, repeated calls, and the chain into gp_build_availability."""
import numpy as np
import pytest

import overhead_ref as ref
from k8s_spark_scheduler_b200 import overhead as oh
from test_overhead_model import _hand_cluster, _random_cluster, both, pod

pytestmark = pytest.mark.gpu

GI = 1 << 30


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def as_lists(triple):
    return tuple(list(map(int, c)) for c in triple)


def check(packer, enc, want=None):
    """device == evaluator (== the restatement's (overhead, nonsched, warned) when given) -> the device's answer"""
    d_ov, d_ns, d_has, d_warned = packer.node_overhead(enc)
    e_ov, e_ns, e_has, e_warned = oh.evaluate(enc)
    assert as_lists(d_ov) == as_lists(e_ov)
    assert as_lists(d_ns) == as_lists(e_ns)
    assert np.array_equal(d_has, e_has)
    assert d_warned == e_warned
    if want is not None:
        assert (as_lists(d_ov), as_lists(d_ns), d_warned) == want
    return d_ov, d_ns, d_has, d_warned


def test_hand_derived(packer):
    pods, lister, rrs, soft = _hand_cluster()
    want, _, enc, has = both(pods, lister, rrs, soft, ["n1", "n2"])
    _, _, d_has, _ = check(packer, enc, want)
    assert d_has.tolist() == [0, 1, 0, 0, 1, 0, 0, 0, 0]


@pytest.mark.parametrize("seed", range(24))
def test_random_string_clusters(packer, seed):
    rng = np.random.default_rng(100 + seed)
    pods, lister, rrs, soft, nodes, events = _random_cluster(rng, 1 + seed % 9, 3 + 13 * seed)
    want, _, enc, _ = both(pods, lister, rrs, soft, nodes, events)
    check(packer, enc, want)


def restated(nodes, lister, rrs, soft, pods):
    comp = ref.OverheadComputer()
    for p in pods:
        comp.on_add(p)
    ov, ns, warned = comp.get_overhead_by_node(nodes, lister, rrs, soft)
    return ref.columns(nodes, ov), ref.columns(nodes, ns), warned


@pytest.mark.parametrize("n_nodes,n_pods,big,huge", [(300, 20_000, 3, 0), (10_000, 300_000, 20, 0), (50_000, 1_000_000, 40, 100_000)])
def test_synthetic_clusters(packer, n_nodes, n_pods, big, huge):
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(n_nodes, n_nodes, n_pods, big_apps=big, huge_app=huge)
    enc = oh.encode(rec.slots, lister, rrs, soft, nodes)
    want = restated(nodes, lister, rrs, soft, pods)
    _, _, has, warned = check(packer, enc, want)
    assert warned > 0 and 0 < has.sum() < n_pods
    if huge:                                              # the 100 000-executor application: 3/4 reserved in its RR
        first = next(i for i, s in enumerate(rec.slots) if s and s[1] == "app-0-exec-0")
        assert 0.97 * (3 * huge) // 4 <= has[first:first + huge].sum() <= (3 * huge) // 4   # less the lister-absent 1 %


def test_listed_nodes_in_any_order_and_subsets(packer):
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(3, 400, 8000, big_apps=2, big_executors=500)
    full = check(packer, oh.encode(rec.slots, lister, rrs, soft, nodes))
    rng = np.random.default_rng(0)
    pick = rng.choice(len(nodes), 150, replace=False)
    part = check(packer, oh.encode(rec.slots, lister, rrs, soft, [nodes[i] for i in pick]))
    for a, b in zip(part[0] + part[1], full[0] + full[1]):
        assert np.array_equal(a, b[pick])


def test_free_slots(packer):
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(5, 100, 3000)
    for p in pods[::3]:
        rec.delete(p)
    comp = ref.OverheadComputer()
    for p in pods:
        comp.on_add(p)
    for p in pods[::3]:
        comp.on_delete(p)
    ov, ns, warned = comp.get_overhead_by_node(nodes, lister, rrs, soft)
    enc = oh.encode(rec.slots, lister, rrs, soft, nodes)
    assert (enc["node_id"] == -1).sum() == len(pods[::3])
    # what a free slot holds is never read
    free = enc["node_id"] == -1
    for k in ("app_key", "app_id", "name_id"):
        enc[k][free] = 1 << 30
    enc["req_cpu_milli"][free] = -5
    check(packer, enc, (ref.columns(nodes, ov), ref.columns(nodes, ns), warned))


def tiny(values, spark=0):
    """pods on node 0 with these cpu requests, no labels -> encoded arrays (one listed node)"""
    n = len(values)
    return dict(n_pods=n, n_node_ids=1, n_app_keys=1, n_app_ids=1, n_names=max(n, 1), node_id=np.zeros(n, np.int32),
                req_cpu_milli=np.array(values, np.int64), req_mem_bytes=np.zeros(n, np.int64), req_gpu=np.array(values, np.int64),
                listed=np.ones(n, np.uint8), app_key=np.full(n, -1, np.int32), app_id=np.full(n, -1, np.int32),
                name_id=np.arange(n, dtype=np.int32), is_executor=np.zeros(n, np.uint8), spark_scheduler=np.full(n, spark, np.uint8),
                n_rr=0, rr_app_key=np.zeros(0, np.int32), rr_pod_off=np.zeros(1, np.int64), rr_pod_name=np.zeros(0, np.int32),
                n_soft=0, soft_app_id=np.zeros(0, np.int32), soft_pod_off=np.zeros(1, np.int64), soft_pod_name=np.zeros(0, np.int32),
                node_ids=np.zeros(1, np.int32))


def test_sums_just_below_and_at_2_61(packer, gangpack):
    top = (1 << 61) - 1
    for vals in ([top], [1 << 60, (1 << 60) - 1], [(1 << 32) - 1] * 1000 + [top - 1000 * ((1 << 32) - 1)],
                 [(1 << 61) // 4096] * 4095 + [(1 << 61) // 4096 - 1]):
        ov, ns, _, _ = check(packer, tiny(vals))
        assert int(ov[0][0]) == int(ns[2][0]) == sum(vals) == top
    for vals in ([1 << 60, 1 << 60], [(1 << 61) // 4096] * 4096, [top, 1]):
        with pytest.raises(gangpack.GangpackError, match="sum >= 2\\^61") as ei:
            packer.node_overhead(tiny(vals, spark=1))              # the overhead alone reaches it
        assert ei.value.status == 6
    with pytest.raises(gangpack.GangpackError, match="request >= 2\\^61") as ei:
        packer.node_overhead(tiny([1 << 61]))
    assert ei.value.status == 6


def small():
    pods, lister, rrs, soft = _hand_cluster()
    rec = oh.PodRecords()
    for p in pods:
        rec.add(p)
    return oh.encode(rec.slots, lister, {**rrs, ("c", "app2"): ["q"]}, {**soft, "app3": ["r"]}, ["n1", "n2"])


REFUSALS = [
    ("negative n_names", lambda e: e.update(n_names=-1), "negative sizes"),
    ("negative n_pods", lambda e: e.update(n_pods=-1), "negative sizes"),
    ("node id out of range", lambda e: e["node_id"].__setitem__(0, e["n_node_ids"]), "out of its range"),
    ("node id below -1", lambda e: e["node_id"].__setitem__(0, -2), "out of its range"),
    ("app key out of range", lambda e: e["app_key"].__setitem__(1, e["n_app_keys"]), "out of its range"),
    ("app id out of range", lambda e: e["app_id"].__setitem__(1, e["n_app_ids"]), "out of its range"),
    ("name out of range", lambda e: e["name_id"].__setitem__(1, e["n_names"]), "out of its range"),
    ("query node out of range", lambda e: e["node_ids"].__setitem__(0, e["n_node_ids"]), "out of its range"),
    ("rr app key out of range", lambda e: e["rr_app_key"].__setitem__(0, -1), "out of its range"),
    ("soft app id out of range", lambda e: e["soft_app_id"].__setitem__(0, e["n_app_ids"]), "out of its range"),
    ("rr pod name out of range", lambda e: e["rr_pod_name"].__setitem__(0, -1), "out of its range"),
    ("soft pod name out of range", lambda e: e["soft_pod_name"].__setitem__(0, e["n_names"]), "out of its range"),
    ("app key without app id", lambda e: e["app_id"].__setitem__(1, -1), "disagree"),
    ("app id without app key", lambda e: e["app_key"].__setitem__(1, -1), "disagree"),
    ("duplicate query node", lambda e: e["node_ids"].__setitem__(1, e["node_ids"][0]), "given twice"),
    ("duplicate rr app key", lambda e: e["rr_app_key"].__setitem__(1, e["rr_app_key"][0]), "given twice"),
    ("duplicate soft app id", lambda e: e["soft_app_id"].__setitem__(1, e["soft_app_id"][0]), "given twice"),
    ("rr offsets not from 0", lambda e: e["rr_pod_off"].__setitem__(0, 1), "does not start at 0"),
    ("soft offsets decrease", lambda e: e["soft_pod_off"].__setitem__(2, 1), "does not start at 0 or decreases"),
    ("negative request", lambda e: e["req_mem_bytes"].__setitem__(2, -1), "negative request"),
    ("negative gpu request", lambda e: e["req_gpu"].__setitem__(6, -1), "negative request"),
]


@pytest.mark.parametrize("name,mutate,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals(packer, gangpack, name, mutate, msg):
    enc = small()
    check(packer, enc)
    mutate(enc)
    with pytest.raises(gangpack.GangpackError, match=msg) as ei:
        packer.node_overhead(enc)
    assert ei.value.status == 1


def test_lister_absent_record_ignores_the_pod_fields(packer):
    enc = small()
    gone = int(np.nonzero(enc["listed"] == 0)[0][0])
    enc["app_key"][gone] = enc["n_app_keys"] + 5
    enc["name_id"][gone] = -7
    check(packer, enc)


def test_empty_inputs(packer):
    enc = tiny([])
    enc["node_ids"] = np.zeros(0, np.int32)
    ov, ns, has, warned = packer.node_overhead(enc)
    assert len(ov[0]) == 0 and len(has) == 0 and warned == 0
    enc = tiny([])
    ov, _, _, _ = packer.node_overhead(enc)
    assert as_lists(ov) == ([0], [0], [0])


def test_context_left_untouched_and_repeatable(packer):
    from k8s_spark_scheduler_b200 import synth
    import k8s_spark_scheduler_b200 as g
    nodes = synth.make_nodes(256, groups=1)
    apps = synth.make_apps(64, groups=1, young_frac=0.0)
    eoff, eorder = synth.group_orders(nodes)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group", "young")}
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    before = packer.pack_batch(a, g.TIGHTLY_PACK, g.MODE_INDEPENDENT)
    stats = packer.stats()
    snap = packer.get_snapshot()
    names, rec, lister, rrs, soft, _ = oh.synthetic_cluster(11, 2000, 60_000, big_apps=4)
    enc = oh.encode(rec.slots, lister, rrs, soft, names)
    first = packer.node_overhead(enc)
    for _ in range(3):
        again = packer.node_overhead(enc)
        assert all(np.array_equal(x, y) for x, y in zip(first[0] + first[1], again[0] + again[1]))
        assert np.array_equal(first[2], again[2]) and first[3] == again[3]
    with pytest.raises(g.GangpackError):
        packer.node_overhead(tiny([-1]))
    assert packer.stats() == stats
    assert all(np.array_equal(x, y) for x, y in zip(packer.get_snapshot(), snap))
    after = packer.pack_batch(a, g.TIGHTLY_PACK, g.MODE_INDEPENDENT)
    assert all(np.array_equal(x, y) for x, y in zip(before, after))


def test_chain_into_build_availability(packer):
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(13, 3000, 60_000, big_apps=3)
    n = len(nodes)
    rng = np.random.default_rng(2)
    alloc = (rng.integers(64, 129, n).astype(np.int64) * 1000, rng.integers(256, 513, n).astype(np.int64) * GI,
             rng.integers(0, 9, n).astype(np.int64))
    res_node = rng.integers(-1, n, 5000).astype(np.int32)
    res = (rng.integers(0, 4000, 5000).astype(np.int64), rng.integers(0, 8, 5000).astype(np.int64) * GI, np.zeros(5000, np.int64))
    d_ov, _, _, _ = packer.node_overhead(oh.encode(rec.slots, lister, rrs, soft, nodes))
    r_ov, _, _ = restated(nodes, lister, rrs, soft, pods)
    r_ov = tuple(np.array(c, np.int64) for c in r_ov)
    got = packer.build_availability(alloc, d_ov, res_node, res)
    want = packer.build_availability(alloc, r_ov, res_node, res)
    assert all(np.array_equal(x, y) for x, y in zip(got[0] + got[1], want[0] + want[1]))
    assert any(np.any(x != y) for x, y in zip(got[0], packer.build_availability(alloc, None, res_node, res)[0]))
