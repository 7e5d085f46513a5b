"""The resident label table (gp_label_table_reset / _update) and the resident affinity entries
(gp_match_node_affinity_resident, gp_exceeds_cluster_capacity_affinity_label_table).

After every flush of affinity.LabelTable, the resident match must equal gp_match_node_affinity on the mirror's decoded labels
bit for bit -- member, n_match, n_error and the status -- and the marker entry must equal
gp_exceeds_cluster_capacity_affinity_resident on the same labels.  Checked over random node-event streams (values that parse
and do not, the int64 limits and one past them, keys added and removed), node tables that permute, subset or repeat the
table's nodes, programs larger than shared memory, every refusal of an update or a query (the table unchanged after it), and
one full-size cluster."""
import numpy as np
import pytest

import capacity_ref as cr
from k8s_spark_scheduler_b200 import affinity as aff
from k8s_spark_scheduler_b200 import native
from test_gpu_exceeds_capacity import make_drivers, make_nodes
from test_gpu_node_affinity import id_cluster
from test_label_table_model import random_cluster, step
from test_overhead_table_model import Driver as OverheadDriver, churn as overhead_churn

pytestmark = pytest.mark.gpu

INVALID = 1
BP = {p: i for i, p in enumerate(cr.PACKERS)}
PROG_KEYS = ("n_aff", "sel_off", "sel_key", "sel_val", "has_required", "term_off", "term_req_off", "term_parse_error", "req_op",
             "req_key", "req_int", "req_val_off", "req_val")


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def outcome(fn):
    try:
        r = fn()
        return 0, tuple(np.asarray(x).tolist() for x in r)
    except native.GangpackError as e:
        return e.status, None


def pair(p, t, ids, progs):
    """(per-call on the mirror's labels, resident) match outcomes for the node table ids"""
    enc = dict(t.to_node_labels(ids), **progs)
    return outcome(lambda: p.match_node_affinity(enc)), outcome(lambda: p.match_node_affinity_resident(ids, progs))


def node_tables(rng, t, live):
    ids = t.node_ids(live)
    perm = rng.permutation(ids)
    sub = perm[:max(1, len(perm) // 3)]
    rep = np.concatenate([sub, sub[:5], [-1, -1]]).astype(np.int32)
    return [ids, perm.astype(np.int32), sub.astype(np.int32), rng.permutation(rep).astype(np.int32), np.zeros(0, np.int32)]


NO_PROGRAMS = dict(n_aff=0, sel_off=np.zeros(1, np.int64), term_off=np.zeros(1, np.int64), term_req_off=np.zeros(1, np.int64),
                   req_val_off=np.zeros(1, np.int64), has_required=np.zeros(0, np.uint8))


def id_programs(rng, t, n, n_aff, big_every=0):
    z = t.mirror.size
    enc = id_cluster(rng, n, n_aff, max_labels=1, n_keys=z["n_keys"], n_values=z["n_values"], big_every=big_every)
    return {k: enc[k] for k in PROG_KEYS}


@pytest.mark.parametrize("seed", range(4))
def test_event_streams(packer, seed):
    rng = np.random.default_rng(seed)
    t = aff.LabelTable(n_node_ids=4, max_labels=2, n_keys=4, n_values=4)
    live, serial = [], [0]
    checked = 0
    for s in range(10):
        step(rng, t, live, serial)
        t.flush(packer)
        _, affs = random_cluster(rng, 1, 20)
        affs.append({"required": [{"matchExpressions": [("ghost", "DoesNotExist", []), ("zone", "NotIn", ["ghost"])]}]})
        for ids in node_tables(rng, t, live):
            names = [f"x{i}" for i in range(len(ids))]
            progs = t.encode_affinities(affs, names)
            for progs in (progs, id_programs(rng, t, len(ids), 12), NO_PROGRAMS):
                a, b = pair(packer, t, ids, progs)
                assert a == b and a[0] == 0, (seed, s)
                checked += 1
    assert checked == 150


def test_int64_limits_and_keys_added_and_removed(packer):
    t = aff.LabelTable()
    vals = ["9223372036854775807", "-9223372036854775808", "9223372036854775808", "-9223372036854775809", "12", "x", "+5", "-0"]
    for i, v in enumerate(vals):
        t.set_node(f"n{i}", {"v": v, f"only{i}": "a"})
    t.flush(packer)
    names = [f"n{i}" for i in range(len(vals))]
    affs = [{"required": [{"matchExpressions": [("v", op, [b])]}]} for op in ("Gt", "Lt") for b in ("0", "9223372036854775806", "5")]
    affs += [{"required": [{"matchExpressions": [(f"only{i}", "Exists", [])]}]} for i in range(3)]
    ids = t.node_ids(names)
    progs = t.encode_affinities(affs, names)
    a, b = pair(packer, t, ids, progs)
    assert a == b and a[0] == 0
    want = aff.evaluate(dict(t.to_node_labels(ids), **progs))
    assert np.array_equal(np.asarray(b[1][0], np.uint32), want[1])
    for i in range(3):                                          # remove the only* keys, add others
        t.set_node(f"n{i}", {"v": vals[i], "new": "b"})
    t.flush(packer)
    a2, b2 = pair(packer, t, ids, t.encode_affinities(affs, names))
    assert a2 == b2 and a2[0] == 0 and b2 != b


def test_programs_larger_than_shared_memory_and_name_fields(packer):
    rng = np.random.default_rng(7)
    t = aff.LabelTable()
    live, serial = [], [0]
    for _ in range(30):
        step(rng, t, live, serial)
    t.flush(packer)
    ids = t.node_ids(live)
    progs = id_programs(rng, t, len(ids), 9, big_every=3)           # ~30 terms x 40 requirements: past 16 KiB
    assert progs["req_op"].size * 16 > 16 * 1024 and (progs["req_op"] >= aff.FIELD_NAME_IN).any()
    a, b = pair(packer, t, ids, progs)
    assert a == b and a[0] == 0


def update_refusals(t):
    """deltas the library must refuse, as (delta, what)"""
    z = t.mirror.size
    ok = dict(row_node=np.array([0], np.int32), row_off=np.array([0, 2], np.int64), label_key=np.array([1, 2], np.int32),
              label_val=np.array([1, 1], np.int32), value_id=np.array([1], np.int32), value_int_ok=np.array([1], np.uint8),
              value_int=np.array([5], np.int64))
    bad = [dict(ok, row_node=np.array([z["n_node_ids"]], np.int32)), dict(ok, row_node=np.array([-1], np.int32)),
           dict(ok, row_node=np.array([0, 0], np.int32), row_off=np.array([0, 1, 2], np.int64)),
           dict(ok, value_id=np.array([1, 1], np.int32), value_int_ok=np.array([1, 1], np.uint8), value_int=np.array([5, 5], np.int64)),
           dict(ok, value_id=np.array([z["n_values"]], np.int32)),
           dict(ok, row_off=np.array([0, z["max_labels"] + 1], np.int64),
                label_key=np.arange(1, z["max_labels"] + 2, dtype=np.int32), label_val=np.ones(z["max_labels"] + 1, np.int32)),
           dict(ok, label_key=np.array([2, 1], np.int32)), dict(ok, label_key=np.array([1, 1], np.int32)),
           dict(ok, label_key=np.array([1, z["n_keys"]], np.int32)), dict(ok, label_val=np.array([1, z["n_values"]], np.int32)),
           dict(ok, label_val=np.array([1, -1], np.int32)), dict(ok, row_off=np.array([1, 2], np.int64))]
    return bad


def test_refusals_leave_the_table_as_it_was(packer, gangpack):
    rng = np.random.default_rng(11)
    t = aff.LabelTable()
    live, serial = [], [0]
    for _ in range(6):
        step(rng, t, live, serial)
    t.flush(packer)
    ids = t.node_ids(live)
    _, affs = random_cluster(rng, 1, 16)
    progs = t.encode_affinities(affs, live)
    before = pair(packer, t, ids, progs)
    assert before[0] == before[1] and before[0][0] == 0
    for k, d in enumerate(update_refusals(t)):
        with pytest.raises(native.GangpackError) as ei:
            packer.label_table_update(d)
        assert ei.value.status == INVALID, k
        assert pair(packer, t, ids, progs) == before, k
    z = t.mirror.size
    with pytest.raises(native.GangpackError):
        packer.label_table_reset(-1, 4, 4, 4)
    with pytest.raises(native.GangpackError):
        packer.label_table_reset(1 << 16, 1 << 15, 4, 4)                    # 2^31 entries
    assert pair(packer, t, ids, progs) == before
    # query refusals
    for bad_ids in (np.array([-2], np.int32), np.array([z["n_node_ids"]], np.int32)):
        assert outcome(lambda: packer.match_node_affinity_resident(bad_ids, progs))[0] == INVALID
    for key, v in (("req_key", z["n_keys"]), ("req_val", z["n_values"]), ("sel_key", z["n_keys"])):
        p2 = id_programs(rng, t, len(ids), 8)
        if p2[key].size == 0:
            continue
        p2[key] = p2[key].copy()
        p2[key][-1] = v
        if key == "req_key":
            p2["req_op"] = np.zeros_like(p2["req_op"])
        assert outcome(lambda: packer.match_node_affinity_resident(ids, p2))[0] == INVALID, key
    name = {"required": [{"matchFields": [("metadata.name", "In", [live[-1]])]}]}
    p3 = t.encode_affinities([name], live)
    assert outcome(lambda: packer.match_node_affinity_resident(ids[:-1], p3))[0] == INVALID  # index past n_nodes
    assert pair(packer, t, ids, progs) == before
    fresh = gangpack.GangPacker()
    try:
        assert outcome(lambda: fresh.match_node_affinity_resident(ids, progs))[0] == INVALID
        with pytest.raises(native.GangpackError) as ei:
            fresh.label_table_update(dict(row_node=np.zeros(0, np.int32)))
        assert ei.value.status == INVALID
    finally:
        fresh.close()


@pytest.mark.parametrize("name", cr.PACKERS)
def test_marker_equals_affinity_resident(packer, name):
    rng = np.random.default_rng(100 + BP[name])
    n, n_zones, q = 80, 3, 120
    t = aff.LabelTable(n_node_ids=8, max_labels=4)
    live, serial = [], [0]
    while len(live) < n:
        step(rng, t, live, serial)
    names = live[:n]
    alloc, _, zone, _ = make_nodes(rng, n, n_zones, 1)
    odrv = OverheadDriver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
    exceeded = fitted = 0
    for s, od in enumerate(overhead_churn(rng, odrv, n - 4, steps=4, per_step=12)):
        odrv.table.push(packer, od)
        for nm in rng.choice(names, 6, replace=False):                 # relabels: keys dropped, a zone set
            kept = dict(list(t.labels[str(nm)].items())[:3])
            t.set_node(str(nm), dict(kept, zone=str(rng.integers(0, 3))))
        t.flush(packer)
        _, affs = random_cluster(rng, 1, 6)
        progs = t.encode_affinities(affs, names)
        ids = t.node_ids(names)
        oids = odrv.table.node_ids(names)
        apps = make_drivers(rng, q, 6, cls_lo=0)
        apps["count"] = rng.integers(0, 6, q).astype(np.int32)
        enc = dict(t.to_node_labels(ids), **progs)
        a = outcome(lambda: packer.exceeds_cluster_capacity_affinity_resident(alloc, oids, enc, apps, BP[name], zone_id=zone, n_zones=n_zones))
        b = outcome(lambda: packer.exceeds_cluster_capacity_affinity_label_table(alloc, oids, ids, progs, apps, BP[name], zone_id=zone,
                                                                              n_zones=n_zones))
        assert a == b and a[0] == 0, (name, s)
        ex, err = np.asarray(a[1][0]), np.asarray(a[1][1])
        exceeded += int(ex[err == 0].sum())
        fitted += int((ex[err == 0] == 0).sum())
    assert exceeded and fitted


def test_full_size(packer):
    """50 000 nodes x 60 labels, 512 affinities"""
    rng = np.random.default_rng(5)
    n, L, A = 50_000, 60, 512
    t = aff.LabelTable(n_node_ids=n, max_labels=L, n_keys=256, n_values=4096)
    keys = [f"k{i}" for i in range(200)]
    for i in range(n):
        ks = rng.choice(200, L, replace=False)
        t.set_node(f"node-{i}", {keys[k]: str(int(v)) if v % 3 else f"v{v}" for k, v in zip(ks, rng.integers(0, 600, L))})
    t.flush(packer)
    ids = t.node_ids([f"node-{i}" for i in range(n)])
    progs = id_programs(rng, t, n, A)
    a, b = pair(packer, t, ids, progs)
    assert a == b and a[0] == 0 and sum(a[1][1]) > 0
