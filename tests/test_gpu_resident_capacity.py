"""gp_exceeds_cluster_capacity_resident and gp_exceeds_cluster_capacity_affinity_resident: the unschedulable-pod marker with
GetNonSchedulableOverhead from the resident overhead table.

Each must return what its per-call entry returns with overhead = gp_overhead_table_query's nonsched_* (zero for a node
without an overhead-table id), bit for bit with the same status: every packer, with and without affinities, over random
overhead event streams; plus each refusal of its own and a per-node sum at 2^61 - 1 and at 2^61."""
import numpy as np
import pytest

import capacity_ref as cr
from k8s_spark_scheduler_b200 import native
from test_gpu_exceeds_capacity import make_drivers, make_nodes
from test_gpu_node_affinity import id_cluster
from test_overhead_table_model import Driver as OverheadDriver, churn as overhead_churn

pytestmark = pytest.mark.gpu

BP = {p: i for i, p in enumerate(cr.PACKERS)}
INVALID, UNREPRESENTABLE = 1, 6


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def outcome(fn):
    try:
        r = fn()
        return 0, [x.tolist() for x in r] if isinstance(r, tuple) else r.tolist()
    except native.GangpackError as e:
        return e.status, None


def pairs(p, names, odrv, alloc, zone, n_zones, group, n_groups, apps, enc, packer_id):
    """[(per-call, resident)] for the node_group form and, with enc, the affinity form"""
    oids = odrv.table.node_ids(names)
    nonsched = odrv.table.answer(names, p.overhead_table_query)[1]
    out = [(outcome(lambda: p.exceeds_cluster_capacity(alloc, apps, packer_id, overhead=nonsched, zone_id=zone, n_zones=n_zones,
                                                       node_group=group, n_groups=n_groups)),
            outcome(lambda: p.exceeds_cluster_capacity_resident(alloc, oids, apps, packer_id, zone_id=zone, n_zones=n_zones,
                                                                node_group=group, n_groups=n_groups)))]
    if enc is not None:
        out.append((outcome(lambda: p.exceeds_cluster_capacity_affinity(alloc, enc, apps, packer_id, overhead=nonsched, zone_id=zone,
                                                                        n_zones=n_zones)),
                    outcome(lambda: p.exceeds_cluster_capacity_affinity_resident(alloc, oids, enc, apps, packer_id, zone_id=zone,
                                                                                 n_zones=n_zones))))
    return out


@pytest.mark.parametrize("name", cr.PACKERS)
def test_random_overhead_streams(packer, name):
    rng = np.random.default_rng(BP[name])
    n, n_zones, n_groups, q, n_aff = 60, 3, 4, 80, 5
    names = [f"n{i}" for i in range(n)]
    alloc, _, zone, group = make_nodes(rng, n, n_zones, n_groups)
    enc = id_cluster(rng, n, n_aff, max_labels=6, n_keys=8, n_values=4)
    odrv = OverheadDriver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
    exceeded = fitted = 0
    for s, od in enumerate(overhead_churn(rng, odrv, n - 4, steps=6, per_step=12)):
        odrv.table.push(packer, od)
        apps = make_drivers(rng, q, n_groups)
        apps["count"] = rng.integers(0, 6, q).astype(np.int32)
        aff_apps = dict(apps, group=rng.integers(0, n_aff, q).astype(np.int32))
        for k, (a, b) in enumerate(pairs(packer, names, odrv, alloc, zone, n_zones, group, n_groups, apps, None, BP[name]) +
                                   pairs(packer, names, odrv, alloc, zone, n_zones, None, 1, aff_apps, enc, BP[name])[1:]):
            assert a[0] == 0 and a == b, (name, s, k)
            ex = a[1] if k == 0 else a[1][0]
            exceeded += sum(ex)
            fitted += len(ex) - sum(ex)
    assert exceeded and fitted and odrv.replays >= 1


def test_without_zones_or_groups_and_no_nodes(packer):
    rng = np.random.default_rng(9)
    names = [f"n{i}" for i in range(20)]
    alloc, _, _, _ = make_nodes(rng, 20, 1, 1)
    odrv = OverheadDriver()
    for od in overhead_churn(rng, odrv, 18, steps=2, per_step=20):
        odrv.table.push(packer, od)
    apps = make_drivers(rng, 30, 1, cls_lo=0)
    for a, b in pairs(packer, names, odrv, alloc, None, 1, None, 1, apps, None, 0):
        assert a[0] == 0 and a == b
    empty = [np.zeros(0, np.int64)] * 3
    a = outcome(lambda: packer.exceeds_cluster_capacity(empty, apps, 0))
    b = outcome(lambda: packer.exceeds_cluster_capacity_resident(empty, None, apps, 0))
    assert a == b and a[1] == [1] * 30                                   # no node: every driver exceeds


def test_refusals_and_sums_at_the_domain_edge(gangpack):
    p = gangpack.GangPacker()
    try:
        rng = np.random.default_rng(23)
        n = 12
        alloc = [np.full(n, 64_000, np.int64), np.full(n, 1 << 40, np.int64), np.zeros(n, np.int64)]
        apps = make_drivers(rng, 10, 1, cls_lo=0)
        oids = np.arange(n, dtype=np.int32)
        run = lambda ids, a=apps: outcome(lambda: p.exceeds_cluster_capacity_resident(alloc, ids, a, 0))[0]
        assert run(oids) == INVALID                                           # no overhead table
        p.overhead_table_reset(n_slots=8, n_node_ids=16, n_app_keys=1, n_app_ids=1, n_names=1)
        assert run(oids) == 0
        assert run(None) == INVALID                                           # overhead_node_id missing
        bad = [np.where(oids == 3, 16, oids), np.where(oids == 3, -2, oids), np.where(oids == 3, 4, oids)]
        for ids in bad:                                                       # out of range (both sides), given twice
            assert run(ids.astype(np.int32)) == INVALID
        negative = dict(apps, exe_cpu=np.where(np.arange(10) == 0, -1, apps["exe_cpu"]))
        assert run(oids, negative) == INVALID                                 # a per-call refusal still applies
        enc = id_cluster(rng, n, 2, max_labels=3, n_keys=4, n_values=4)
        aff_apps = dict(apps, group=rng.integers(0, 2, 10).astype(np.int32))
        assert outcome(lambda: p.exceeds_cluster_capacity_affinity_resident(alloc, bad[2].astype(np.int32), enc, aff_apps, 0))[0] == INVALID
        # two records on node id 15 summing to 2^61 - 1 (a result), then to 2^61 (refused by both entries)
        for top, want in (((1 << 60) - 1, 0), (1 << 60, UNREPRESENTABLE)):
            p.overhead_table_update(dict(slot=[0, 1], node_id=[15, 15], req_cpu_milli=[1 << 60, top], req_mem_bytes=[0, 0],
                                         listed=[1, 1], app_key=[-1, -1], app_id=[-1, -1], name_id=[0, 0]))
            ids = np.where(oids == 5, 15, oids).astype(np.int32)
            got = [run(ids), outcome(lambda: p.exceeds_cluster_capacity_affinity_resident(alloc, ids, enc, aff_apps, 0))[0]]
            assert got == [want, want], top
            if want == 0:
                q = p.overhead_table_query(ids[5:6], has_reservation=False)[1]
                assert q[0][0] == (1 << 61) - 1
                nonsched = [np.where(oids == 5, int(q[d][0]), 0).astype(np.int64) for d in range(3)]
                same = lambda: p.exceeds_cluster_capacity(alloc, apps, 0, overhead=nonsched)
                assert outcome(same) == outcome(lambda: p.exceeds_cluster_capacity_resident(alloc, ids, apps, 0))
    finally:
        p.close()


def test_full_size(packer):
    """50 000 nodes, 1 000 000 overhead records, 1 000 stale drivers, every packer"""
    rng = np.random.default_rng(50_000)
    n, n_zones, n_groups, q = 50_000, 3, 8, 1000
    alloc, _, zone, group = make_nodes(rng, n, n_zones, n_groups)
    recs = 1_000_000
    slot = np.arange(recs, dtype=np.int32)
    p = packer
    p.overhead_table_reset(n_slots=recs, n_node_ids=n, n_app_keys=1, n_app_ids=1, n_names=1)
    node = rng.integers(0, n, recs).astype(np.int32)
    cpu, mem = rng.integers(0, 500, recs), rng.integers(0, 1 << 28, recs)
    spark = (rng.random(recs) < 0.5).astype(np.uint8)
    p.overhead_table_update(dict(slot=slot, node_id=node, req_cpu_milli=cpu, req_mem_bytes=mem, listed=np.ones(recs, np.uint8),
                                 app_key=np.full(recs, -1, np.int32), app_id=np.full(recs, -1, np.int32),
                                 name_id=np.zeros(recs, np.int32), spark_scheduler=spark))
    oids = rng.permutation(n).astype(np.int32)                            # node-table entry i carries overhead id oids[i]
    nonsched = p.overhead_table_query(oids, has_reservation=False)[1]
    apps = make_drivers(rng, q, n_groups)
    apps["count"] = rng.integers(0, 400, q).astype(np.int32)
    for name in cr.PACKERS:
        a = outcome(lambda: p.exceeds_cluster_capacity(alloc, apps, BP[name], overhead=nonsched, zone_id=zone, n_zones=n_zones,
                                                       node_group=group, n_groups=n_groups))
        b = outcome(lambda: p.exceeds_cluster_capacity_resident(alloc, oids, apps, BP[name], zone_id=zone, n_zones=n_zones,
                                                                node_group=group, n_groups=n_groups))
        assert a[0] == 0 and a == b, name
