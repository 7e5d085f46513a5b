"""gp_match_node_affinity and gp_exceeds_cluster_capacity_affinity on the device.

The match is checked bit for bit against the string oracle (tests/affinity_ref.py) on small clusters and against the numpy
evaluator of the encoded programs (itself checked against the oracle on CPU) up to 50 000 nodes and 512 affinities, including
programs too large for shared memory.  The capacity check over overlapping affinity sets is checked against
capacity_ref.literal_exceeds / the T + M criterion over each driver's matched nodes, against gp_exceeds_cluster_capacity on
disjoint affinities, and across affinity chunks."""
import numpy as np
import pytest

import affinity_ref as ar
import capacity_ref as cr
from k8s_spark_scheduler_b200 import affinity as aff
from test_affinity_model import random_cluster, term

pytestmark = pytest.mark.gpu

GI = 1 << 30
BP = {p: i for i, p in enumerate(cr.PACKERS)}


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


# ---- synthetic clusters given directly as ids (large) ---------------------------------------------------------------------
def id_cluster(rng, n, n_aff, max_labels=40, n_keys=48, n_values=24, big_every=0):
    """nodes with 0..max_labels labels over n_keys keys; n_aff random programs over the same ids"""
    cnt = rng.integers(0, max_labels + 1, n)
    off = np.zeros(n + 1, np.int64); np.cumsum(cnt, out=off[1:])
    keys = np.concatenate([np.sort(rng.choice(n_keys, c, replace=False)) for c in cnt]).astype(np.int32) if n else np.zeros(0, np.int32)
    vals = rng.integers(0, n_values, len(keys)).astype(np.int32)
    ok = (rng.random(len(keys)) < 0.7).astype(np.uint8)
    ival = np.where(ok, rng.integers(-20, 20, len(keys)), 0).astype(np.int64)
    sel_off, sel_key, sel_val, has_req, term_off = [0], [], [], [], [0]
    tro, terr, op, rk, ri, rvo, rv = [0], [], [], [], [], [0], []
    for a in range(n_aff):
        if rng.random() < 0.2:
            ks = rng.choice(n_keys, int(rng.integers(1, 3)), replace=False)
            sel_key += ks.tolist(); sel_val += rng.integers(0, 4, len(ks)).tolist()
        sel_off.append(len(sel_key))
        has_req.append(rng.random() > 0.1)
        big = big_every and a % big_every == 0
        for _ in range(int(rng.integers(0, 4)) if not big else 30):
            terr.append(int(rng.random() < 0.05))
            for _ in range(int(rng.integers(0, 4)) if not big else 40):
                o = int(rng.integers(0, 8))
                op.append(o); rk.append(int(rng.integers(0, n_keys)))
                ri.append(int(rng.integers(-1, n)) if o >= 6 else int(rng.integers(-10, 10)))
                if o in (0, 1):
                    rv += np.sort(rng.choice(n_values, min(n_values, int(rng.integers(1, 6 if not big else 20))), replace=False)).tolist()
                rvo.append(len(rv))
            tro.append(len(op))
        term_off.append(len(terr))
    i32, i64, u8 = (lambda x: np.asarray(x, np.int32)), (lambda x: np.asarray(x, np.int64)), (lambda x: np.asarray(x, np.uint8))
    return dict(n_nodes=n, n_keys=n_keys, n_values=n_values, n_aff=n_aff, label_off=off, label_key=keys, label_val=vals,
                label_int_ok=ok, label_int=ival, sel_off=i64(sel_off), sel_key=i32(sel_key), sel_val=i32(sel_val),
                has_required=u8(has_req), term_off=i64(term_off), term_req_off=i64(tro), term_parse_error=u8(terr),
                req_op=i32(op), req_key=i32(rk), req_int=i64(ri), req_val_off=i64(rvo), req_val=i32(rv))


def check_match(packer, enc):
    member, n_match, n_error = packer.match_node_affinity(enc)
    _, w_member, w_match, w_error = aff.evaluate(enc)
    assert np.array_equal(member, w_member)
    assert np.array_equal(n_match, w_match) and np.array_equal(n_error, w_error)
    return member, n_match, n_error


# ---- match ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_match_equals_string_oracle(packer, seed):
    rng = np.random.default_rng(100 + seed)
    nodes, affs = random_cluster(rng, int(rng.integers(1, 300)), int(rng.integers(1, 60)))
    enc = aff.encode(nodes, affs)
    member, n_match, n_error = packer.match_node_affinity(enc)
    want = np.array([[ar.outcome(p, nd) for nd in nodes] for p in affs], np.int8)
    assert np.array_equal(aff.unpack_bits(member, len(nodes)), want == 1)
    assert np.array_equal(n_match, (want == 1).sum(1)) and np.array_equal(n_error, (want == 2).sum(1))


def test_match_reference_quirks(packer):
    nodes = [{"name": "n0", "labels": {"zone": "a", "gpus": "8"}}, {"name": "n1", "labels": {"zone": "b", "gpus": "x"}},
             {"name": "n2", "labels": {}}]
    affs = [{"required": []},                                                         # empty required affinity: nothing
            {"required": [term(("gpus", "NotIn", ["8"]))]},                           # NotIn on an absent key matches
            {"nodeSelector": {"zone": "a"}, "required": [term(("zone", "Bogus", []))]},  # selector masks the parse error
            {"required": [term(("zone", "In", [])), term(("zone", "In", ["a"]))]},   # error only where no term matched
            {"required": [term(("gpus", "Gt", ["4"]))]},                              # non-integer node value: no match
            {"required": [term(fields=[("metadata.name", "In", ["n1"])])]},
            {"required": [term(fields=[("metadata.name", "NotIn", ["ghost"])])]},
            {"required": None}]
    member, n_match, n_error = packer.match_node_affinity(aff.encode(nodes, affs))
    got = aff.unpack_bits(member, 3).astype(int).tolist()
    assert got == [[0, 0, 0], [0, 1, 1], [0, 0, 0], [1, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 1], [1, 1, 1]]
    assert n_error.tolist() == [0, 0, 1, 2, 0, 0, 0, 0]


@pytest.mark.parametrize("n,n_aff", [(1, 1), (33, 7), (10_000, 16), (10_000, 128), (50_000, 512)])
def test_match_large_random(packer, n, n_aff):
    rng = np.random.default_rng(n + n_aff)
    check_match(packer, id_cluster(rng, n, n_aff))


def oversized_cluster(rng, n, n_aff, V=8):
    """Every node carries keys 0..9 (values 0..V-1, key 9 an integer); key 20 is on no node.  Affinity a (every third one
    larger than shared memory: 30 terms x 40 requirements) has terms of requirements that hold on every node -- In with all
    values, Exists, NotIn on the absent key, DoesNotExist on it, Gt below every integer -- plus one selective In with a
    single value, so each term matches a different part of the cluster and later terms decide what earlier ones did not."""
    off = np.arange(n + 1, dtype=np.int64) * 10
    keys = np.tile(np.arange(10, dtype=np.int32), n)
    vals = rng.integers(0, V, 10 * n).astype(np.int32)
    ok = (keys == 9).astype(np.uint8)
    ival = np.where(ok, rng.integers(0, 100, 10 * n), 0).astype(np.int64)
    sel_off, term_off, tro, terr, op, rk, ri, rvo, rv = [0], [0], [0], [], [], [], [], [0], []
    for a in range(n_aff):
        sel_off.append(0)
        big = a % 3 == 0
        for t in range(30 if big else 2):
            terr.append(0)
            m = 40 if big else 3
            sel = int(rng.integers(0, m))
            for r in range(m):
                if r == sel:                                                # the selective requirement
                    o, k, vs, b = 0, int(rng.integers(0, 9)), [int(rng.integers(0, V))], 0
                else:
                    kind = r % 5
                    o, k, vs, b = [(0, r % 9, list(range(V)), 0), (2, r % 10, [], 0), (1, 20, [0, 1], 0), (3, 20, [], 0),
                                   (4, 9, [], -1)][kind]
                op.append(o); rk.append(k); ri.append(b); rv += vs; rvo.append(len(rv))
            tro.append(len(op))
        term_off.append(len(terr))
    i32, i64, u8 = (lambda x: np.asarray(x, np.int32)), (lambda x: np.asarray(x, np.int64)), (lambda x: np.asarray(x, np.uint8))
    return dict(n_nodes=n, n_keys=21, n_values=V, n_aff=n_aff, label_off=off, label_key=keys, label_val=vals, label_int_ok=ok,
                label_int=ival, sel_off=i64(sel_off), sel_key=i32([]), sel_val=i32([]), has_required=u8([1] * n_aff),
                term_off=i64(term_off), term_req_off=i64(tro), term_parse_error=u8(terr), req_op=i32(op), req_key=i32(rk),
                req_int=i64(ri), req_val_off=i64(rvo), req_val=i32(rv))


def test_match_programs_larger_than_shared_memory(packer):
    rng = np.random.default_rng(7)
    enc = oversized_cluster(rng, 3000, 24)
    reqs = np.diff(enc["term_req_off"][enc["term_off"]])
    vals = np.diff(enc["req_val_off"][enc["term_req_off"][enc["term_off"]]])
    big = 24 * reqs + 4 * vals > 16 * 1024                   # at least 24 bytes per requirement and 4 per value id
    assert big.sum() == 8
    member, n_match, n_error = check_match(packer, enc)
    # the oversized programs decide by their requirements: partial matches, no errors
    assert (n_error[big] == 0).all() and (n_match[big] > 0).all() and (n_match[big] < 3000).all()
    # and their later terms matter: the first term alone matches fewer nodes
    first_only = {**enc, "term_parse_error": enc["term_parse_error"].copy()}
    for a in np.nonzero(big)[0]:                             # mark every term after the first as a parse error
        first_only["term_parse_error"][enc["term_off"][a] + 1:enc["term_off"][a + 1]] = 1
    m1, n1, e1 = check_match(packer, first_only)
    assert (n1[big] < n_match[big]).all() and (e1[big] > 0).all()


# ---- capacity over overlapping affinity sets ------------------------------------------------------------------------------
def overlap_cluster(rng, n, n_zones):
    """labels: ig (4 groups), zone, node type; affinities that overlap: by ig, ig + zone, ig In several, none at all"""
    ig, zone = rng.integers(0, 4, n), rng.integers(0, n_zones, n)
    typ = rng.choice(["cpu", "gpu", "mem"], n)
    nodes = [{"name": f"n{i}", "labels": {"ig": f"g{ig[i]}", "zone": f"z{zone[i]}", "type": str(typ[i])}} for i in range(n)]
    affs = [{"required": None}]
    affs += [{"nodeSelector": {"ig": f"g{k}"}} for k in range(4)]
    affs += [{"required": [term(("ig", "In", [f"g{k}"]), ("zone", "In", [f"z{z}"]))]} for k in range(4) for z in range(min(n_zones, 2))]
    affs += [{"required": [term(("ig", "In", ["g0", "g1", "g2"]))]}, {"required": [term(("type", "NotIn", ["gpu"]))]},
             {"required": [term(("ig", "In", ["g3"])), term(("type", "In", ["gpu"]))]}, {"required": []},
             {"required": [term(("zone", "In", ["bad value"]))]},                                    # an error on every node
             {"nodeSelector": {"ig": "g1"}, "required": [term(("zone", "In", ["bad value"]))]}]     # error on g1 only
    return nodes, affs, zone.astype(np.int32)


def node_quantities(rng, n):
    from test_gpu_exceeds_capacity import make_nodes
    alloc, over, _, _ = make_nodes(rng, n, 1, 1)
    return alloc, over


def driver_batch(rng, q, n_aff, sets, alloc, over, zone, n_zones):
    from test_gpu_exceeds_capacity import make_drivers, shapes
    apps = make_drivers(rng, q, n_aff, cls_lo=0)
    sched = [alloc[d] - over[d] for d in range(3)]
    for i in range(q):                            # counts at the T + M boundary of the driver's own matched set
        drv, exe = shapes(apps, i)
        m = sets[int(apps["group"][i])]
        T, M = cr.np_zone_terms([s[m] for s in sched], zone[m], n_zones, drv, exe)
        fit = M > cr.NONE
        b = int(T.sum()) + int(M[fit].max()) if fit.any() else None
        r = rng.random()
        k = int(rng.integers(0, 20)) if b is None or r < 0.15 else (b + 1 if r < 0.5 else b - int(rng.integers(0, 3)))
        apps["count"][i] = max(0, min(k, (1 << 31) - 1))
    return apps


def model(name, apps, sets, alloc, over, zone, n_zones):
    from test_gpu_exceeds_capacity import shapes
    sched = [alloc[d] - over[d] for d in range(3)]
    out = np.zeros(len(apps["count"]), np.uint8)
    for i in range(len(out)):
        drv, exe = shapes(apps, i)
        m = sets[int(apps["group"][i])]
        T, M = cr.np_zone_terms([s[m] for s in sched], zone[m], n_zones, drv, exe)
        out[i] = cr.np_decide(name, T, M, drv, exe, int(apps["count"][i]))
    return out


@pytest.mark.parametrize("name", cr.PACKERS)
@pytest.mark.parametrize("n,n_zones", [(40, 1), (300, 3), (5000, 5)])
def test_capacity_overlapping_sets(packer, name, n, n_zones):
    rng = np.random.default_rng(n + n_zones + BP[name])
    nodes, affs, zone = overlap_cluster(rng, n, n_zones)
    enc = aff.encode(nodes, affs)
    outcome = aff.evaluate(enc)[0]
    sets = [np.nonzero(outcome[a] == 1)[0] for a in range(len(affs))]
    assert np.mean((outcome == 1).sum(0)) > 2                     # most nodes are in several affinities
    alloc, over = node_quantities(rng, n)
    apps = driver_batch(rng, 300, len(affs), sets, alloc, over, zone, n_zones)
    got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, BP[name], overhead=over, zone_id=zone, n_zones=n_zones)
    want_err = (outcome == 2).any(1)[apps["group"]]
    assert np.array_equal(err.astype(bool), want_err)
    ok = ~want_err
    assert np.array_equal(got[ok], model(name, apps, sets, alloc, over, zone, n_zones)[ok])
    # the literal marker on a slice
    names = [nd["name"] for nd in nodes]
    A = {names[i]: tuple(int(alloc[d][i]) for d in range(3)) for i in range(n)}
    O = {names[i]: tuple(int(over[d][i]) for d in range(3)) for i in range(n)}
    Zl = {names[i]: f"zone-{zone[i]}" for i in range(n)}
    from test_gpu_exceeds_capacity import shapes
    for i in rng.choice(np.nonzero(ok)[0], 30 if n <= 300 else 4, replace=False):
        drv, exe = shapes(apps, i)
        k = int(apps["count"][i])
        if k > 4096:
            continue
        order = [names[j] for j in sets[int(apps["group"][i])]]
        assert cr.literal_exceeds(name, A, O, Zl, order, drv, exe, k) == bool(got[i]), (i, k)


@pytest.mark.parametrize("name", cr.PACKERS)
def test_disjoint_affinities_equal_node_group_call(packer, name):
    rng = np.random.default_rng(11 + BP[name])
    n, n_zones = 4000, 4
    ig = rng.integers(-1, 6, n)                                   # -1: a node without the label
    zone = rng.integers(0, n_zones, n).astype(np.int32)
    nodes = [{"name": f"n{i}", "labels": {"ig": f"g{ig[i]}"} if ig[i] >= 0 else {}} for i in range(n)]
    affs = [{"nodeSelector": {"ig": f"g{k}"}} for k in range(6)]
    enc = aff.encode(nodes, affs)
    alloc, over = node_quantities(rng, n)
    sets = [np.nonzero(ig == k)[0] for k in range(6)]
    apps = driver_batch(rng, 500, 6, sets, alloc, over, zone, n_zones)
    got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, BP[name], overhead=over, zone_id=zone, n_zones=n_zones)
    want = packer.exceeds_cluster_capacity(alloc, apps, BP[name], overhead=over, zone_id=zone, n_zones=n_zones,
                                           node_group=ig.astype(np.int32), n_groups=6)
    assert not err.any()
    assert np.array_equal(got, want)


def test_affinity_chunks_equal_hand_split(packer):
    # 600 affinities over 20 000 nodes: K = 2^21 / 20 000 = 104 affinities per chunk, six chunks
    rng = np.random.default_rng(5)
    n, n_aff = 20_000, 600
    enc = id_cluster(rng, n, n_aff, max_labels=12, n_keys=16, n_values=4)
    enc["term_parse_error"][:] = 0
    alloc, over = node_quantities(rng, n)
    from test_gpu_exceeds_capacity import make_drivers
    apps = make_drivers(rng, 3000, n_aff, cls_lo=0)
    apps["count"] = rng.integers(0, 3000, 3000).astype(np.int32)
    for name in ("tightly-pack", "single-az-tightly-pack"):
        got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, BP[name], overhead=over)
        # by hand: one call per block of 50 affinities, each with only its own affinities and drivers
        want, werr = np.zeros_like(got), np.zeros_like(err)
        for a0 in range(0, n_aff, 50):
            sub = sub_affinities(enc, a0, min(a0 + 50, n_aff))
            idx = np.nonzero((apps["group"] >= a0) & (apps["group"] < a0 + 50))[0]
            part = {k: (v[idx] if isinstance(v, np.ndarray) else v) for k, v in apps.items()}
            part["group"] = part["group"] - a0
            want[idx], werr[idx] = packer.exceeds_cluster_capacity_affinity(alloc, sub, part, BP[name], overhead=over)
        assert np.array_equal(err, werr) and np.array_equal(got[err == 0], want[err == 0])


def sub_affinities(enc, a0, a1):
    """the programs of affinities [a0, a1) as an encoding of their own (same labels)"""
    out = {k: v for k, v in enc.items()}
    t0, t1 = enc["term_off"][a0], enc["term_off"][a1]
    r0, r1 = enc["term_req_off"][t0], enc["term_req_off"][t1]
    v0, v1 = enc["req_val_off"][r0], enc["req_val_off"][r1]
    s0, s1 = enc["sel_off"][a0], enc["sel_off"][a1]
    out.update(n_aff=a1 - a0, sel_off=enc["sel_off"][a0:a1 + 1] - s0, sel_key=enc["sel_key"][s0:s1], sel_val=enc["sel_val"][s0:s1],
               has_required=enc["has_required"][a0:a1], term_off=enc["term_off"][a0:a1 + 1] - t0,
               term_req_off=enc["term_req_off"][t0:t1 + 1] - r0, term_parse_error=enc["term_parse_error"][t0:t1],
               req_op=enc["req_op"][r0:r1], req_key=enc["req_key"][r0:r1], req_int=enc["req_int"][r0:r1],
               req_val_off=enc["req_val_off"][r0:r1 + 1] - v0, req_val=enc["req_val"][v0:v1])
    return out


# ---- refusals, untouched context, empty batches ---------------------------------------------------------------------------
def small():
    nodes = [{"name": "a", "labels": {"k": "1"}}, {"name": "b", "labels": {"k": "2", "m": "x"}}]
    return aff.encode(nodes, [{"required": [term(("k", "In", ["1", "2"]))]}, {"nodeSelector": {"m": "x"}}])


@pytest.mark.parametrize("case,msg", [
    (lambda e: e.update(label_off=np.array([1, 1, 3])), "label_off"),
    (lambda e: e.update(label_off=np.array([0, 2, 1])), "label_off"),
    (lambda e: e["label_key"].__setitem__(1, 99), "label key"),
    (lambda e: e.update(label_key=e["label_key"][[0, 2, 1]].copy()), "label key"),
    (lambda e: e["label_val"].__setitem__(0, -1), "label value"),
    (lambda e: e["req_op"].__setitem__(0, 8), "operator"),
    (lambda e: e["req_key"].__setitem__(0, 77), "key id"),
    (lambda e: e.update(req_val=e["req_val"][::-1].copy()), "strictly ascending"),
    (lambda e: e["req_val"].__setitem__(0, 500), "value id"),
    (lambda e: e["sel_val"].__setitem__(0, 500), "selector"),
    (lambda e: (e["req_op"].__setitem__(0, 6), e["req_int"].__setitem__(0, 2)), "metadata.name"),
    (lambda e: e.update(term_off=np.array([0, 2, 1])), "term_off"),
])
def test_refusals(packer, gangpack, case, msg):
    enc = small()
    case(enc)
    with pytest.raises(gangpack.GangpackError) as ei:
        packer.match_node_affinity(enc)
    assert ei.value.status == 1 and msg in str(ei.value) and "gp_match_node_affinity" in str(ei.value)
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI])]
    apps = dict(drv_cpu=[0], drv_mem=[0], exe_cpu=[1000], exe_mem=[GI], count=[1], group=[0])
    with pytest.raises(gangpack.GangpackError) as ei:
        packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, 0)
    assert ei.value.status == 1 and msg in str(ei.value)
    packer.match_node_affinity(small())                         # a valid call right after succeeds


def test_capacity_refusals_and_empty_batch(packer, gangpack):
    enc = small()
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI])]
    apps = dict(drv_cpu=[0, 0], drv_mem=[0, 0], exe_cpu=[1000, 1000], exe_mem=[GI, GI], count=[16, 9], group=[0, 1])
    got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, 0)
    assert got.tolist() == [0, 1] and err.tolist() == [0, 0]
    for bad in ([2, 0], [-1, 0]):
        with pytest.raises(gangpack.GangpackError, match="driver group out of range"):
            packer.exceeds_cluster_capacity_affinity(alloc, enc, dict(apps, group=bad), 0)
    with pytest.raises(gangpack.GangpackError, match="unknown packer"):
        packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, 9)
    empty = dict(drv_cpu=[], drv_mem=[], exe_cpu=[], exe_mem=[], count=[], group=[])
    got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, empty, 0)
    assert len(got) == 0
    with pytest.raises(gangpack.GangpackError, match="allocatable"):       # an empty batch still validates the nodes
        packer.exceeds_cluster_capacity_affinity([np.array([1 << 62, 0]), alloc[1]], enc, empty, 0)
    with pytest.raises(gangpack.GangpackError, match="zone_id"):
        packer.exceeds_cluster_capacity_affinity(alloc, enc, empty, 0, zone_id=np.array([0, 3], np.int32), n_zones=2)


def test_no_affinities(packer, gangpack):
    """zero programs: the match returns nothing and the capacity call succeeds on an empty batch; the labels and nodes are
    still checked"""
    nodes = [{"name": "a", "labels": {"k": "1"}}, {"name": "b", "labels": {"k": "2"}}]
    enc = aff.encode(nodes, [])
    member, n_match, n_error = packer.match_node_affinity(enc)
    assert member.shape[0] == 0 and len(n_match) == 0 and len(n_error) == 0
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI])]
    empty = dict(drv_cpu=[], drv_mem=[], exe_cpu=[], exe_mem=[], count=[], group=[])
    got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, empty, 0)
    assert len(got) == 0
    with pytest.raises(gangpack.GangpackError, match="driver group out of range"):
        packer.exceeds_cluster_capacity_affinity(alloc, enc, dict(drv_cpu=[0], drv_mem=[0], exe_cpu=[0], exe_mem=[0], count=[0],
                                                                  group=[0]), 0)
    bad = dict(enc, label_val=np.array([0, 7], np.int32))
    for call in (lambda: packer.match_node_affinity(bad), lambda: packer.exceeds_cluster_capacity_affinity(alloc, bad, empty, 0)):
        with pytest.raises(gangpack.GangpackError, match="label value id out of range"):
            call()
    with pytest.raises(gangpack.GangpackError, match="allocatable"):
        packer.exceeds_cluster_capacity_affinity([np.array([1 << 62, 0]), alloc[1]], enc, empty, 0)


def test_context_left_untouched(packer):
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
    rng = np.random.default_rng(1)
    nodes2, affs, zone = overlap_cluster(rng, 500, 3)
    alloc, over = node_quantities(rng, 500)
    enc = aff.encode(nodes2, affs)
    packer.match_node_affinity(enc)
    packer.exceeds_cluster_capacity_affinity(alloc, enc, dict(drv_cpu=[1000], drv_mem=[GI], exe_cpu=[1000], exe_mem=[GI],
                                                              count=[3], group=[2]), 2, overhead=over, zone_id=zone, n_zones=3)
    assert packer.stats() == stats
    assert all(np.array_equal(x, y) for x, y in zip(packer.get_snapshot(), snap))
    after = packer.pack_batch(a, g.TIGHTLY_PACK, g.MODE_INDEPENDENT)
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
