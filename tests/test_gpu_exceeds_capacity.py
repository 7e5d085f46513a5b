"""gp_exceeds_cluster_capacity: the unschedulable-pod marker's sweep on the device, every packer.

Checked against the literal DoesPodExceedClusterCapacity (tests/capacity_ref.py over oracle/pyref.py), the restated
criterion, and the existing entry points on the same inputs; plus counts above 2^24, a 50 000-node / 100 000-driver sweep,
the untouched context and every refusal."""
import numpy as np
import pytest

import capacity_ref as cr
import fingerprint_ref as fr
from k8s_spark_scheduler_b200 import affinity as aff

pytestmark = pytest.mark.gpu

GI = 1 << 30
BP = {p: i for i, p in enumerate(cr.PACKERS)}


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def make_nodes(rng, n, n_zones, n_groups):
    ac = rng.integers(1, 65, n) * 1000 + np.where(rng.random(n) < 0.3, rng.integers(0, 1000, n), 0)
    am = rng.integers(1, 257, n) * GI + np.where(rng.random(n) < 0.2, rng.integers(0, 1 << 20, n), 0)
    ag = np.where(rng.random(n) < 0.3, rng.integers(1, 9, n), 0)
    oc = np.where(rng.random(n) < 0.5, rng.integers(0, 2000, n), 0)
    om = np.where(rng.random(n) < 0.5, rng.integers(0, 2 * GI, n), 0)
    og = np.where(rng.random(n) < 0.05, ag + 1, 0)                       # a negative schedulable gpu
    neg = rng.random(n) < 0.03
    oc = np.where(neg, ac + 1000, oc)                                     # negative schedulable cpu
    f = lambda x: np.asarray(x, np.int64)
    zone = rng.integers(0, n_zones, n).astype(np.int32)
    group = rng.integers(-1, n_groups, n).astype(np.int32)
    return [f(ac), f(am), f(ag)], [f(oc), f(om), f(og)], zone, group


def make_drivers(rng, q, n_groups, gpus=True, cls_lo=-1):
    dc = rng.choice([0, 500, 1000, 2000, 4000], q); dm = rng.choice([0, GI, 2 * GI, 4 * GI], q)
    ec = rng.choice([0, 1, 500, 1000, 2000, 8000], q); em = rng.choice([0, GI // 2, GI, 4 * GI, 16 * GI], q)
    dg = np.where(rng.random(q) < (0.2 if gpus else 0), rng.integers(0, 3, q), 0)
    eg = np.where(rng.random(q) < (0.2 if gpus else 0), rng.integers(0, 3, q), 0)
    f = lambda x: np.asarray(x, np.int64)
    return dict(drv_cpu=f(dc), drv_mem=f(dm), drv_gpu=f(dg), exe_cpu=f(ec), exe_mem=f(em), exe_gpu=f(eg),
                group=rng.integers(cls_lo, n_groups, q).astype(np.int32), count=np.zeros(q, np.int32))


def shapes(apps, i):
    return ((int(apps["drv_cpu"][i]), int(apps["drv_mem"][i]), int(apps["drv_gpu"][i])),
            (int(apps["exe_cpu"][i]), int(apps["exe_mem"][i]), int(apps["exe_gpu"][i])))


def members(group, cls):
    return np.arange(len(group)) if cls == -1 else np.nonzero(group == cls)[0]


def class_terms(alloc, over, zone, n_zones, group, apps, cache=None):
    """{(class, drv, exe): (T[z], M[z])} for every driver of the batch (vectorised criterion, one entry per distinct tuple)"""
    sched = [alloc[d] - over[d] for d in range(3)]
    cache = {} if cache is None else cache
    for i in range(len(apps["count"])):
        drv, exe = shapes(apps, i)
        key = (int(apps["group"][i]), drv, exe)
        if key not in cache:
            m = members(group, key[0])
            cache[key] = cr.np_zone_terms([s[m] for s in sched], zone[m], n_zones, drv, exe)
    return cache


def model_all(name, apps, cache):
    out = np.zeros(len(apps["count"]), np.uint8)
    for i in range(len(out)):
        drv, exe = shapes(apps, i)
        T, M = cache[(int(apps["group"][i]), drv, exe)]
        out[i] = cr.np_decide(name, T, M, drv, exe, int(apps["count"][i]))
    return out


def set_counts_around_boundary(rng, apps, cache, frac_exceed=1 / 3):
    """count = T + M (fits) or T + M + 1 (exceeds) over the whole class, plus some small counts"""
    for i in range(len(apps["count"])):
        drv, exe = shapes(apps, i)
        T, M = cache[(int(apps["group"][i]), drv, exe)]
        fit = M > cr.NONE
        b = int(T.sum()) + int(M[fit].max()) if fit.any() else None
        r = rng.random()
        if b is None or r < 0.15:
            k = int(rng.integers(0, 20))
        elif r < 0.15 + frac_exceed:
            k = b + 1
        else:
            k = b - int(rng.integers(0, 3))
        apps["count"][i] = max(0, min(k, (1 << 31) - 1))


def call(packer, alloc, over, zone, n_zones, group, n_groups, apps, name):
    return packer.exceeds_cluster_capacity(alloc, apps, BP[name], overhead=over, zone_id=zone, n_zones=n_zones,
                                           node_group=group, n_groups=n_groups)


# ---- the reference's own scenarios ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", cr.PACKERS)
def test_reference_marker_scenarios(packer, name):
    # TestUnschedulablePodMarker / TestSchedulerFailsToScheduleWhenNotEnoughNvidiaGPUs: two 8 CPU / 8 GiB / 1 GPU nodes in
    # zone1; the driver asks 1 CPU, 1 byte, 1 GPU, executors 1 CPU and 1 byte (and 1 GPU)
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI]), np.array([1, 1])]
    apps = dict(drv_cpu=[1000] * 3, drv_mem=[1] * 3, drv_gpu=[1] * 3, exe_cpu=[1000] * 3, exe_mem=[1] * 3, exe_gpu=[0, 0, 1],
                count=[2, 100, 2], group=[0, 0, 0])
    got = packer.exceeds_cluster_capacity(alloc, apps, BP[name])
    assert got.tolist() == [0, 1, 1]


# ---- random clusters against the literal marker -----------------------------------------------------------------------
@pytest.mark.parametrize("name", cr.PACKERS)
@pytest.mark.parametrize("n,n_groups,n_zones", [(30, 1, 1), (60, 3, 7), (200, 20, 70), (800, 5, 3), (3000, 20, 12)])
def test_random_clusters_against_literal(packer, name, n, n_groups, n_zones):
    rng = np.random.default_rng(n * 31 + n_groups * 7 + n_zones + BP[name])
    alloc, over, zone, group = make_nodes(rng, n, n_zones, n_groups)
    q = 400
    apps = make_drivers(rng, q, n_groups)
    cache = class_terms(alloc, over, zone, n_zones, group, apps)
    set_counts_around_boundary(rng, apps, cache)
    got = call(packer, alloc, over, zone, n_zones, group, n_groups, apps, name)
    want = model_all(name, apps, cache)
    assert np.array_equal(got, want)
    assert 0 < want.sum() < q
    # the literal path on a slice (pure-Python packers: the node count sets the slice)
    names = [f"node-{i}" for i in range(n)]
    A = {names[i]: (int(alloc[0][i]), int(alloc[1][i]), int(alloc[2][i])) for i in range(n)}
    O = {names[i]: (int(over[0][i]), int(over[1][i]), int(over[2][i])) for i in range(n)}
    Zl = {names[i]: f"zone-{zone[i]}" for i in range(n)}
    for i in rng.choice(q, 40 if n <= 200 else 6, replace=False):
        drv, exe = shapes(apps, i)
        k = int(apps["count"][i])
        if k > 4096 or (n > 800 and apps["group"][i] < 0):      # the literal packers loop once per executor
            continue
        order = [names[j] for j in members(group, int(apps["group"][i]))]
        rng.shuffle(order)
        assert cr.literal_exceeds(name, A, O, Zl, order, drv, exe, k) == bool(got[i]), (i, drv, exe, k)


def test_empty_class_and_no_nodes(packer):
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI]), None]
    apps = dict(drv_cpu=[0, 0, 0], drv_mem=[0, 0, 0], exe_cpu=[0, 0, 0], exe_mem=[0, 0, 0], count=[0, 0, 5], group=[1, -1, 0])
    for name in cr.PACKERS:
        got = packer.exceeds_cluster_capacity(alloc, apps, BP[name], node_group=np.array([0, 0], np.int32), n_groups=2)
        sa = name.startswith("single-az")                # an all-zero application has no positive efficiency
        assert got.tolist() == [1, 1 if sa else 0, 1 if sa else 0]
        empty = [np.zeros(0, np.int64)] * 2 + [None]
        assert packer.exceeds_cluster_capacity(empty, apps, BP[name], n_groups=2).tolist() == [1, 1, 1]


# ---- counts above 2^24 ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", cr.PACKERS)
def test_counts_above_2_24(packer, name):
    rng = np.random.default_rng(24 + BP[name])
    n, n_zones = 2000, 4
    alloc = [rng.integers(32, 129, n) * 1000, rng.integers(64, 513, n) * GI, np.zeros(n, np.int64)]
    over = [np.zeros(n, np.int64)] * 3
    zone = rng.integers(0, n_zones, n).astype(np.int32)
    group = np.zeros(n, np.int32)
    q = 64
    apps = dict(drv_cpu=np.full(q, 1000), drv_mem=np.full(q, GI), drv_gpu=np.zeros(q, np.int64),
                exe_cpu=rng.choice([0, 1, 2, 3], q).astype(np.int64), exe_mem=rng.choice([0, 1, 4096], q).astype(np.int64),
                exe_gpu=np.zeros(q, np.int64), group=np.zeros(q, np.int32), count=np.zeros(q, np.int32))
    cache = class_terms(alloc, over, zone, n_zones, group, apps)
    set_counts_around_boundary(rng, apps, cache, frac_exceed=0.5)
    apps["count"][:4] = [(1 << 31) - 1, 1 << 25, (1 << 24) + 1, 1 << 30]
    assert (apps["count"] > (1 << 24)).sum() >= 10
    got = call(packer, alloc, over, zone, n_zones, group, 1, apps, name)
    want = model_all(name, apps, cache)
    assert np.array_equal(got, want)


# ---- 50 000 nodes, 16 classes x 8 zones, 100 000 drivers --------------------------------------------------------------
def test_fullsize_sweep(packer):
    rng = np.random.default_rng(50_000)
    n, n_groups, n_zones, q = 50_000, 16, 8, 100_000
    alloc, over, zone, group = make_nodes(rng, n, n_zones, n_groups)
    apps = make_drivers(rng, q, n_groups)
    cache = class_terms(alloc, over, zone, n_zones, group, apps)
    set_counts_around_boundary(rng, apps, cache)
    for name in cr.PACKERS:
        got = call(packer, alloc, over, zone, n_zones, group, n_groups, apps, name)
        want = model_all(name, apps, cache)
        assert np.array_equal(got, want), name
        if name == "tightly-pack":
            assert 0.25 < want.mean() < 0.45
    # the literal path on a slice: drivers of small counts in one class
    name = "tightly-pack"
    got = call(packer, alloc, over, zone, n_zones, group, n_groups, apps, name)
    names = [f"node-{i}" for i in range(n)]
    A = {names[i]: (int(alloc[0][i]), int(alloc[1][i]), int(alloc[2][i])) for i in range(n)}
    O = {names[i]: (int(over[0][i]), int(over[1][i]), int(over[2][i])) for i in range(n)}
    Zl = {names[i]: f"zone-{zone[i]}" for i in range(n)}
    picked = [i for i in range(q) if apps["group"][i] >= 0 and apps["count"][i] <= 50 and shapes(apps, i)[1] != (0, 0, 0)][:5]
    for i in picked:
        drv, exe = shapes(apps, i)
        order = [names[j] for j in members(group, int(apps["group"][i]))]
        assert cr.literal_exceeds(name, A, O, Zl, order, drv, exe, int(apps["count"][i])) == bool(got[i])


# ---- agreement with the existing entry points -------------------------------------------------------------------------
def _cluster_for_entries(seed, n=600, n_groups=4, n_zones=5, q=600):
    rng = np.random.default_rng(seed)
    alloc, over, zone, group = make_nodes(rng, n, n_zones, n_groups)
    apps = make_drivers(rng, q, n_groups, cls_lo=0)
    set_counts_around_boundary(rng, apps, class_terms(alloc, over, zone, n_zones, group, apps))
    apps["count"] = np.minimum(apps["count"], 1 << 20).astype(np.int32)
    sched = [alloc[d] - over[d] for d in range(3)]
    return rng, alloc, over, zone, group, apps, sched


@pytest.mark.parametrize("name,algo", [("tightly-pack", 0), ("distribute-evenly", 1)])
def test_agrees_with_pack_batch(gangpack, name, algo):
    rng, alloc, over, zone, group, apps, sched = _cluster_for_entries(7 + algo)
    n_groups = 4
    aux = gangpack.GangPacker()
    try:
        orders = [rng.permutation(members(group, g)) for g in range(n_groups)]
        off = np.zeros(n_groups + 1, np.int32)
        off[1:] = np.cumsum([len(o) for o in orders])
        order = np.concatenate(orders).astype(np.int32)
        aux.set_snapshot(sched[0], sched[1], sched[2], order, order, off, off)
        drv, _, _ = aux.pack_batch(apps, algo)
        got = call(aux, alloc, over, zone, 5, group, n_groups, apps, name)
        assert np.array_equal(got, (drv < 0).astype(np.uint8))
    finally:
        aux.close()


@pytest.mark.parametrize("name,algo", [("single-az-tightly-pack", 0), ("single-az-minimal-fragmentation", 2)])
def test_agrees_with_pack_batch_zones(gangpack, name, algo):
    rng, alloc, over, zone, group, apps, sched = _cluster_for_entries(11 + algo)
    aux = gangpack.GangPacker()
    try:
        call_all = call(aux, alloc, over, zone, 5, group, 4, apps, name)
        for g in range(4):
            sel = np.nonzero(apps["group"] == g)[0]
            sub = {k: np.asarray(v)[sel] for k, v in apps.items()}
            m = members(group, g)
            zs = [z for z in dict.fromkeys(zone[rng.permutation(m)].tolist())]
            orders = [rng.permutation(m[zone[m] == z]) for z in zs]
            off = np.zeros(len(orders) + 1, np.int32)
            off[1:] = np.cumsum([len(o) for o in orders])
            order = np.concatenate(orders).astype(np.int32)
            aux.set_snapshot(sched[0], sched[1], sched[2], order, order, off, off)
            aux.set_schedulable(sched[0], sched[1], sched[2])
            z, _, _, _, _ = aux.pack_batch_zones(sub, algo)
            assert np.array_equal(call_all[sel], (z < 0).astype(np.uint8)), g
    finally:
        aux.close()


def test_agrees_with_pack_batch_az_aware(gangpack):
    rng, alloc, over, zone, group, apps, sched = _cluster_for_entries(13)
    aux = gangpack.GangPacker()
    try:
        call_all = call(aux, alloc, over, zone, 5, group, 4, apps, "az-aware-tightly-pack")
        for g in range(4):
            sel = np.nonzero(apps["group"] == g)[0]
            sub = {k: np.asarray(v)[sel] for k, v in apps.items()}
            m = members(group, g)
            undivided = rng.permutation(m).astype(np.int32)
            zs = list(dict.fromkeys(zone[undivided].tolist()))
            orders = [undivided[zone[undivided] == z] for z in zs]
            off = np.zeros(len(orders) + 1, np.int32)
            off[1:] = np.cumsum([len(o) for o in orders])
            order = np.concatenate(orders).astype(np.int32)
            aux.set_snapshot(sched[0], sched[1], sched[2], order, order, off, off)
            aux.set_schedulable(sched[0], sched[1], sched[2])
            _, drv, _, _, _ = aux.pack_batch_az_aware(sub, undivided, undivided, len(zs))
            assert np.array_equal(call_all[sel], (drv < 0).astype(np.uint8)), g
    finally:
        aux.close()


# ---- the context is left alone ----------------------------------------------------------------------------------------
def test_context_untouched(gangpack):
    rng, alloc, over, zone, group, apps, sched = _cluster_for_entries(17)
    n = len(zone)
    order = rng.permutation(n).astype(np.int32)
    off = np.array([0, n], np.int32)
    pack_apps = {k: (np.zeros(len(v), np.int32) if k == "group" else v) for k, v in apps.items()}
    a, fresh = gangpack.GangPacker(), gangpack.GangPacker()
    try:
        for p in (a, fresh):
            p.set_snapshot(sched[0], sched[1], sched[2], order, order, off, off)
        before = a.get_snapshot()
        stats_before = a.stats()
        for name in cr.PACKERS:
            call(a, alloc, over, zone, 5, group, 4, apps, name)
        after = a.get_snapshot()
        for x, y in zip(before, after):
            assert np.array_equal(x, y)
        assert a.stats() == stats_before
        r1, r2 = a.pack_batch(pack_apps, 0), fresh.pack_batch(pack_apps, 0)
        for x, y in zip(r1, r2):
            assert np.array_equal(x, y)
    finally:
        a.close(); fresh.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals(gangpack, packer):
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI]), np.array([1, 0])]
    good = dict(drv_cpu=[1000], drv_mem=[GI], exe_cpu=[1000], exe_mem=[GI], count=[1], group=[0])
    zone = np.array([0, 1], np.int32)
    grp = np.array([0, -1], np.int32)

    def run(apps=good, a=alloc, p=0, **kw):
        kw.setdefault("zone_id", zone); kw.setdefault("n_zones", 2); kw.setdefault("node_group", grp); kw.setdefault("n_groups", 1)
        return packer.exceeds_cluster_capacity(a, apps, p, **kw)

    assert run().tolist() == [0]
    cases = [
        (dict(apps=dict(good, drv_cpu=[-1])), 1, "negative"),
        (dict(apps=dict(good, exe_mem=[-5])), 1, "negative"),
        (dict(apps=dict(good, count=[-1])), 1, "negative"),
        (dict(apps=dict(good, group=[1])), 1, "driver group"),
        (dict(apps=dict(good, group=[-2])), 1, "driver group"),
        (dict(zone_id=np.array([0, 2], np.int32)), 1, "zone_id"),
        (dict(zone_id=np.array([-1, 0], np.int32)), 1, "zone_id"),
        (dict(node_group=np.array([0, 1], np.int32)), 1, "node_group"),
        (dict(node_group=np.array([-2, 0], np.int32)), 1, "node_group"),
        (dict(p=5), 1, "packer"),
        (dict(p=-1), 1, "packer"),
        (dict(n_groups=0), 1, "n_groups"),
        (dict(n_zones=0), 1, "n_zones"),
        (dict(apps=dict(good, exe_cpu=[1 << 61])), 6, "2\\^61"),
        (dict(apps=dict(good, drv_gpu=[1 << 61])), 6, "2\\^61"),
        (dict(a=[alloc[0], np.array([1 << 61, 0]), alloc[2]]), 6, "allocatable"),
        (dict(a=[np.array([-(1 << 61), 0]), alloc[1], alloc[2]]), 6, "allocatable"),
    ]
    for kw, status, msg in cases:
        with pytest.raises(gangpack.native.GangpackError, match=msg) as e:
            run(**kw)
        assert e.value.status == status, kw
    with pytest.raises(gangpack.native.GangpackError, match="allocatable") as e:
        packer.exceeds_cluster_capacity(alloc, good, 0, overhead=[np.array([0, 1 << 61]), None, None])
    assert e.value.status == 6
    assert run().tolist() == [0]                          # the context still works after every refusal


# ---- interning: drivers whose fingerprints collide -----------------------------------------------------------------------
def test_same_fingerprint_in_one_warp(packer):
    # Rows whose chained fingerprints F(F(F(exe), drv cpu, drv mem), drv gpu, class) collide (tests/fingerprint_ref.py): A
    # fits (answer 0); B (class 0, like A) and C (A's requests in another class) ask for 2^50 or more driver GPUs (answer
    # 1), so a row given another row's pair flips its answer.  A and B interleaved inside warps: the multi-round match loop;
    # in warps and CTAs of their own: a probe passing an entry of equal fingerprint and another tuple.
    A, B, C, ga, gc = fr.marker_rows()
    assert fr.marker_fingerprint(A, 0) == fr.marker_fingerprint(B, 0) and fr.marker_fingerprint(A, ga) == fr.marker_fingerprint(C, gc)
    n_groups = max(ga, gc) + 1
    n = 4 * n_groups
    alloc = [np.full(n, 8000), np.full(n, 8 * GI), np.zeros(n, np.int64)]
    group = (np.arange(n) % n_groups).astype(np.int32)
    zone = np.zeros(n, np.int32)
    nodes = [{"name": f"n{i}", "labels": {"ig": f"g{group[i]}"}} for i in range(n)]
    enc = aff.encode(nodes, [{"nodeSelector": {"ig": f"g{k}"}} for k in range(n_groups)])
    within = [(A, 0) if i % 3 else (B, 0) for i in range(96)]
    across = [(B, 0) if i // 256 == 0 or (i // 32) % 2 else (A, 0) for i in range(1024)]
    classes = [[(A, ga), (C, gc), (A, gc)][i % 3] for i in range(96)] + [(C, gc)] * 64 + [(A, ga)] * 64
    for rows in (within, across, classes):
        cols = list(zip(*[r for r, _ in rows]))
        apps = dict(drv_cpu=cols[0], drv_mem=cols[1], drv_gpu=cols[2], exe_cpu=cols[3], exe_mem=cols[4], exe_gpu=cols[5],
                    count=np.full(len(rows), 3, np.int32), group=np.array([g for _, g in rows], np.int32))
        apps = {k: np.asarray(v) for k, v in apps.items()}
        cache = class_terms(alloc, [np.zeros(n, np.int64)] * 3, zone, 1, group, apps)
        want = [0 if r == A else 1 for r, _ in rows]
        for name in cr.PACKERS:
            assert model_all(name, apps, cache).tolist() == want, name
            assert call(packer, alloc, None, zone, 1, group, n_groups, apps, name).tolist() == want, name
            got, err = packer.exceeds_cluster_capacity_affinity(alloc, enc, apps, BP[name], zone_id=zone)
            assert not err.any() and got.tolist() == want, name


# ---- buckets of more than one segment (4 096 nodes) and one zone per node ----------------------------------------------
@pytest.mark.parametrize("n,n_groups,n_zones", [(30_000, 1, 3), (12_000, 2, 1), (6_000, 2, 6_000)])
def test_large_buckets_and_many_zones(packer, n, n_groups, n_zones):
    rng = np.random.default_rng(n + n_zones)
    alloc, over, zone, group = make_nodes(rng, n, n_zones, n_groups)
    if n_zones == n:
        zone = rng.permutation(n).astype(np.int32)                # one zone per node
    apps = make_drivers(rng, 3000, n_groups)
    cache = class_terms(alloc, over, zone, n_zones, group, apps)
    set_counts_around_boundary(rng, apps, cache)
    for name in cr.PACKERS:
        got = call(packer, alloc, over, zone, n_zones, group, n_groups, apps, name)
        assert np.array_equal(got, model_all(name, apps, cache)), name


def test_empty_batch_still_validates_nodes(gangpack, packer):
    alloc = [np.array([8000, 8000]), np.array([8 * GI, 8 * GI]), None]
    none = dict(drv_cpu=[], drv_mem=[], exe_cpu=[], exe_mem=[], count=[], group=[])
    assert packer.exceeds_cluster_capacity(alloc, none, 0).tolist() == []
    for kw, msg in ((dict(zone_id=np.array([0, 3], np.int32), n_zones=2), "zone_id"),
                    (dict(node_group=np.array([0, 4], np.int32)), "node_group")):
        with pytest.raises(gangpack.native.GangpackError, match=msg) as e:
            packer.exceeds_cluster_capacity(alloc, none, 0, **kw)
        assert e.value.status == 1
    with pytest.raises(gangpack.native.GangpackError, match="allocatable") as e:
        packer.exceeds_cluster_capacity([alloc[0], np.array([1 << 61, 0]), None], none, 0)
    assert e.value.status == 6
