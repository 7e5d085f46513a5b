"""gp_reconcile_find_nodes: the failover reconciler's findNodes loop on the device.

Checked bit for bit (placed, every ExecutorNodes slice, the availability after the loop) against the literal restatements of
tests/reconcile_ref.py -- the string-keyed C literal on random clusters, the pyref literal on small ones -- and against the closed
form at 50 000 nodes; plus the sizes around the kernel's tiles, counts up to 2^24, every refusal and the untouched context."""
import numpy as np
import pytest

import reconcile_ref as R

pytestmark = pytest.mark.gpu

GI = 1 << 30


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def run(p, case, **kw):
    ng, dg, count, G = R.to_device_args(case)
    apps = dict(exe_cpu=case["exe"][0], exe_mem=case["exe"][1], exe_gpu=case["exe"][2], count=count, group=dg)
    return p.reconcile_find_nodes(case["alloc"], case["overhead"], case["res_node"], case["res"], ng, case["creation"], apps,
                                  kw.pop("n_groups", G), unschedulable=case["unschedulable"], ready=case["ready"], **kw)


def check(got, want):
    gp_, go, goff, gav = got
    wp, wo, woff, wav = want[:4]
    assert np.array_equal(goff, woff)
    assert np.array_equal(gp_, wp)
    for i in np.nonzero(wp > 0)[0]:
        s = slice(woff[i], woff[i] + wp[i])
        assert np.array_equal(go[s], wo[s]), i
    for d in range(3):
        assert [int(x) for x in gav[d]] == [int(x) for x in wav[d]], d


def test_random_clusters_against_the_c_literal(packer):
    rng = np.random.default_rng(7)
    for it in range(40):
        n = int(rng.integers(30, 3001))
        case = R.random_case(rng, n, int(rng.integers(1, 71)), int(rng.integers(1, 2001)), int(rng.integers(0, 4 * n)))
        want = R.c_literal(case)
        assert not want[4]
        check(run(packer, case), want)


def test_small_clusters_against_the_pyref_literal(packer):
    rng = np.random.default_rng(11)
    for it in range(300):
        case = R.random_case(rng, int(rng.integers(0, 40)), int(rng.integers(1, 6)), int(rng.integers(0, 14)), int(rng.integers(0, 60)))
        check(run(packer, case), R.literal_flat(case))


def test_every_node_dropped_or_empty_table(packer):
    rng = np.random.default_rng(3)
    case = R.random_case(rng, 50, 3, 40, 80)
    case["ready"] = np.zeros(50, np.uint8)
    got = run(packer, case)
    assert (got[0] == -1).all()
    check(got, R.literal_flat(case))
    empty = R.random_case(rng, 0, 1, 5, 0)
    assert (run(packer, empty)[0] == -1).all()


def _large(rng, n, groups, q, rows):
    case = R.random_case(rng, n, groups, q, rows)
    case["alloc"] = (case["alloc"][0] * 4, case["alloc"][1] * 4, case["alloc"][2])
    big = rng.random(q) < 0.01                    # some drivers ask for more than their group holds
    case["min"] = np.where(big, 50_000, case["min"])
    return case


def test_large_cluster_against_closed_form_and_literal(packer):
    rng = np.random.default_rng(50_000)
    case = _large(rng, 50_000, 64, 10_000, 100_000)
    got = run(packer, case)
    check(got, R.closed_form(case))
    lit = R.c_literal(case)
    check(got, lit)
    _, _, count, _ = R.to_device_args(case)
    assert ((got[0] >= 0) & (got[0] < count)).any()          # partial placements happen


def test_group_larger_than_a_tile_and_more_groups_than_sms(packer):
    rng = np.random.default_rng(5)
    one = R.random_case(rng, 3000, 1, 2000, 6000)              # one group of ~2 400 schedulable nodes: many tiles per walk
    one["min"] = rng.integers(0, 400, 2000)
    check(run(packer, one), R.c_literal(one))
    many = R.random_case(rng, 3000, 200, 2000, 6000)           # 200 groups claimed by the persistent grid
    check(run(packer, many), R.c_literal(many))


def _single_node(cpu, k, exe_cpu=1000, n=1):
    return dict(names=[f"n{i}" for i in range(n)], alloc=(np.full(n, cpu, np.int64), np.full(n, 1 << 50, np.int64), np.zeros(n, np.int64)),
                label=["g"] * n, unschedulable=None, ready=None, creation=np.arange(n, 0, -1).astype(np.int64), overhead=None,
                res_node=np.zeros(0, np.int32), res=(np.zeros(0, np.int64),) * 3, dgroup=["g"] * len(k),
                exe=(np.full(len(k), exe_cpu, np.int64), np.zeros(len(k), np.int64), np.zeros(len(k), np.int64)),
                min=np.array(k, np.int64), running=np.zeros(len(k), np.int64))


@pytest.mark.parametrize("k", [65_535, 65_536, 1 << 24])
def test_large_counts(packer, k):
    case = _single_node(1000 * (k + 3), [k, 5])                # the second driver finds 3 left and overshoots
    got = run(packer, case)
    want = R.closed_form(case)
    check(got, want)
    assert list(got[0]) == [k, 3]
    spread = _single_node(1000 * 7, [k], n=300)                # 7 per node over 300 nodes, the rest unplaced
    check(run(packer, spread), R.closed_form(spread))


def test_count_above_2_24_is_refused(gangpack, packer):
    case = _single_node(1 << 40, [(1 << 24) + 1])
    with pytest.raises(gangpack.native.GangpackError) as e:
        run(packer, case)
    assert e.value.status == 6


def test_domain_exit_through_overshoot_is_refused(gangpack, packer):
    big = (1 << 60) + 7
    case = _single_node(1 << 60, [1, 1, 1], exe_cpu=big)       # each driver overshoots once more: -2^60 - ... - 2^60 leaves 2^61
    assert R.closed_form(case)[4] and R.c_literal(case)[4]
    with pytest.raises(gangpack.native.GangpackError) as e:
        run(packer, case)
    assert e.value.status == 6
    ok = _single_node(1 << 60, [1], exe_cpu=big)                # one overshoot stays inside the domain
    check(run(packer, ok), R.closed_form(ok))


def test_validation_refusals(gangpack, packer):
    rng = np.random.default_rng(9)
    base = R.random_case(rng, 20, 2, 6, 10)
    ng, dg, count, G = R.to_device_args(base)

    def call(node_group=ng, group=dg, cnt=count, exe=base["exe"], n_groups=G, **kw):
        apps = dict(exe_cpu=exe[0], exe_mem=exe[1], exe_gpu=exe[2], count=cnt, group=group)
        return packer.reconcile_find_nodes(base["alloc"], base["overhead"], base["res_node"], base["res"], node_group, base["creation"],
                                           apps, n_groups, **kw)

    def refused(status, **kw):
        with pytest.raises(gangpack.native.GangpackError) as e:
            call(**kw)
        assert e.value.status == status, kw

    refused(1, node_group=np.where(np.arange(20) == 3, G, ng))
    refused(1, node_group=np.where(np.arange(20) == 3, -1, ng))
    refused(1, group=np.where(np.arange(6) == 2, G, dg))
    refused(1, group=np.where(np.arange(6) == 2, -1, dg))
    refused(1, cnt=np.where(np.arange(6) == 1, -1, count))
    refused(1, n_groups=0)
    neg = (np.where(np.arange(6) == 0, -1, base["exe"][0]), base["exe"][1], base["exe"][2])
    refused(1, exe=neg)
    huge = (base["exe"][0], np.where(np.arange(6) == 0, 1 << 61, base["exe"][1]), base["exe"][2])
    refused(6, exe=huge)
    need = int(count.sum())
    if need:
        refused(5, exec_cap=need - 1)
    call()                                                      # the good call still works


def test_context_untouched_and_repeatable(gangpack):
    rng = np.random.default_rng(17)
    case = R.random_case(rng, 800, 8, 500, 2000)
    n = 800
    avail = [np.asarray(x, np.int64) for x in case["alloc"]]
    order = rng.permutation(n).astype(np.int32)
    off = np.array([0, n], np.int32)
    apps = dict(drv_cpu=np.full(50, 1000), drv_mem=np.full(50, GI), drv_gpu=np.zeros(50), exe_cpu=np.full(50, 2000),
                exe_mem=np.full(50, 2 * GI), exe_gpu=np.zeros(50), count=rng.integers(0, 8, 50).astype(np.int32),
                group=np.zeros(50, np.int32), young=np.zeros(50, np.uint8))
    a, fresh = gangpack.GangPacker(), gangpack.GangPacker()
    try:
        for p in (a, fresh):
            p.set_snapshot(avail[0], avail[1], avail[2], order, order, off, off)
        a.pack_batch(apps, 0)
        before, stats_before = a.get_snapshot(), a.stats()
        r1 = run(a, case)
        r2 = run(a, case)
        for x, y in zip(r1[:3], r2[:3]):
            assert np.array_equal(x, y)
        for x, y in zip(r1[3], r2[3]):
            assert np.array_equal(x, y)
        for x, y in zip(before, a.get_snapshot()):
            assert np.array_equal(x, y)
        assert a.stats() == stats_before
        fresh.pack_batch(apps, 0)
        for x, y in zip(a.pack_batch(apps, 0), fresh.pack_batch(apps, 0)):
            assert np.array_equal(x, y)
    finally:
        a.close(); fresh.close()
