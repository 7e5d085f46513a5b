"""gp_reschedule_from_reservations: rescheduleExecutor from the reservations to the node choice in one device call.  Checked
- against the five-call sequence it replaces (gp_build_availability, gp_build_reschedule_availability, gp_potential_nodes,
  gp_set_snapshot, gp_reschedule_executors): node_out bit-identical, both branches, batches of executors;
- the ambiguity flag against the arg-min model of tests/reschedule_ref.py;
- end to end against the literal rescheduleExecutor chain, scopes that drop zones and the missing-label refusal included;
- the context state: a resident driver snapshot (gp_prepare_cluster, FIFO, gp_reserve_placements(subtract)) and an az-aware
  layout (orders == NULL) behave as if the call never happened;
- the launches: no sort kernel, one stream synchronise; edge cases and refusals."""
import numpy as np
import pytest

import reschedule_ref as rr
from helpers import random_apps
from reschedule_ref import ZONE_LABEL
from test_gpu_prepare_zones import make_case, sort_args

pytestmark = pytest.mark.gpu

G = 1 << 30


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


@pytest.fixture(scope="module")
def recipe(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def executors(rng, q, n, hosting=True):
    exe = (rng.integers(0, 9, q) * 250, rng.integers(0, 17, q) * (G // 4), (rng.integers(0, 6, q) == 0).astype(np.int64))
    host = [list(rng.integers(0, n, int(rng.integers(0, 6)))) for _ in range(q)] if hosting else None
    return exe, host


def one_call(p, c, exe, min_frag, host, keep=None, tz=None, labels=True):
    zid, nz, rank, _, unsched, ready, _, lre = sort_args(c)
    return p.reschedule_from_reservations(c["alloc"], c["over"], c["rnode"], c["res"], exe, min_frag=min_frag, hosting=host,
                                          zone_id=zid, n_zones=nz, name_rank=rank, unschedulable=unsched, ready=ready,
                                          executor_label_rank=lre if labels else None, keep_topology_zone=keep, topology_zone=tz)


def five_calls(p, c, exe, min_frag, host, labels=True):
    """What a caller does without the new entry: two availabilities and the order to the host, one snapshot upload."""
    zid, nz, rank, cand, unsched, ready, lrd, lre = sort_args(c)
    meta, _ = p.build_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    ff = p.build_reschedule_availability(c["alloc"], c["over"], c["rnode"], c["res"])
    _, eo = p.potential_nodes(meta[0], meta[1], zid, nz, rank, cand, unsched, ready, lrd, lre if labels else None, avail_gpu=meta[2])
    av = meta if min_frag else ff
    p.set_snapshot(av[0], av[1], av[2], eo, eo)
    got = p.reschedule_executors(exe, min_frag=min_frag, reserved=c["over"] if min_frag else None, hosting=host if min_frag else None)
    return got, meta, ff


def model_flags(c, meta, ff, exe, min_frag, host, labels=True):
    n = len(c["names"])
    zid = c["zid"]
    member = [True] * n
    cand = [not c["unsched"][i] and bool(c["ready"][i]) for i in range(n)]
    tri = lambda a, i: (int(a[0][i]), int(a[1][i]), int(a[2][i]))
    out = []
    for x in range(len(exe[0])):
        e = (int(exe[0][x]), int(exe[1][x]), int(exe[2][x]))
        out.append(rr.decide([tri(meta, i) for i in range(n)], [tri(ff, i) for i in range(n)], [tri(c["over"], i) for i in range(n)],
                             zid, c["rank"], member, cand, c["lre"] if labels else None, e, min_frag,
                             set(int(h) for h in host[x]) if (min_frag and host) else set()))
    return out


@pytest.mark.parametrize("seed,n,Z", [(1, 300, 3), (2, 900, 1), (3, 2500, 8), (4, 5000, 16), (5, 700, 4)])
@pytest.mark.parametrize("min_frag", [False, True])
def test_equals_five_call_sequence(packer, recipe, seed, n, Z, min_frag):
    c = make_case(seed, n, Z)
    rng = np.random.default_rng(seed + 100)
    exe, host = executors(rng, 96, n)
    for labels in (True, False):
        got, amb = one_call(packer, c, exe, min_frag, host, labels=labels)
        want, meta, ff = five_calls(recipe, c, exe, min_frag, host, labels=labels)
        assert np.array_equal(got, want), (seed, labels, np.nonzero(got != want)[0][:5])
        if n <= 900:
            flags = model_flags(c, meta, ff, exe, min_frag, host, labels)
            assert [w for w, _ in flags] == list(got), (seed, labels)
            assert [int(a) for _, a in flags] == list(amb), (seed, labels)


def test_ties_flagged(packer, recipe):
    """equal (memory, cpu) with differing gpu: flagged exactly where the model says; node_out still equals the sequence"""
    n = 400
    rng = np.random.default_rng(11)
    c = make_case(11, n, 2, R=0, labels=False)
    c["alloc"] = [np.full(n, 8000, np.int64), np.full(n, 16 * G, np.int64), rng.integers(0, 3, n).astype(np.int64)]
    c["over"] = [np.zeros(n, np.int64)] * 3
    exe, host = executors(rng, 64, n)
    for mf in (False, True):
        got, amb = one_call(packer, c, exe, mf, host, labels=False)
        want, meta, ff = five_calls(recipe, c, exe, mf, host, labels=False)
        assert np.array_equal(got, want)
        flags = model_flags(c, meta, ff, exe, mf, host, labels=False)
        assert [int(a) for _, a in flags] == list(amb)
        assert amb.any()


def literal_case(seed, n=60, Z=3, missing=0.0):
    rng = np.random.default_rng(seed)
    c = make_case(seed, n, Z, R=n * 2, zone_p=np.ones(Z))
    # the topology label (filterNodesToZone) is drawn independently of the sorter's zone (the beta label, zone_id): the
    # reference reads the two from different labels (SURVEY App. B5)
    c["tz"] = np.where(rng.random(n) < missing, -1, rng.integers(0, Z, n)).astype(np.int32)
    return c


def test_sorter_zone_and_topology_zone_are_separate(packer):
    """a: 8 cores / 8 GiB in topology zone 0; b, c: 6 / 6 in topology zone 1; no beta label, so one sorter zone: the
    reference chooses b.  With the sorter zones equal to the topology zones it chooses a (zone 0 has the smaller totals)."""
    alloc = [np.array([8000, 6000, 6000]), np.array([8, 6, 6]) * G, np.zeros(3, np.int64)]
    tz = np.array([0, 1, 1], np.int32)
    exe = ([1000], [G], [0])
    args = dict(name_rank=np.arange(3, dtype=np.int32))
    got, _ = packer.reschedule_from_reservations(alloc, None, np.zeros(0, np.int32), [np.zeros(0, np.int64)] * 3, exe,
                                                 zone_id=np.zeros(3, np.int32), n_zones=1, **args)
    assert list(got) == [1]
    got, _ = packer.reschedule_from_reservations(alloc, None, np.zeros(0, np.int32), [np.zeros(0, np.int64)] * 3, exe,
                                                 zone_id=tz, n_zones=2, **args)
    assert list(got) == [0]
    got, _ = packer.reschedule_from_reservations(alloc, None, np.zeros(0, np.int32), [np.zeros(0, np.int64)] * 3, exe,
                                                 zone_id=np.zeros(3, np.int32), n_zones=1, keep_topology_zone=1, topology_zone=tz, **args)
    assert list(got) == [1]


def literal_decisions(c, exe, min_frag, host, keep):
    names = c["names"]
    n = len(names)
    tri = lambda a, i: (int(a[0][i]), int(a[1][i]), int(a[2][i]))
    labels = {names[i]: ({ZONE_LABEL: "z%d" % c["tz"][i]} if c["tz"][i] >= 0 else {}) for i in range(n)}
    sort_zone = {names[i]: "z%d" % c["zid"][i] for i in range(n)}
    alloc = {names[i]: tri(c["alloc"], i) for i in range(n)}
    over = {names[i]: tri(c["over"], i) for i in range(n)}
    resv = [(names[r] if r >= 0 else "gone-%d" % t, tri(c["res"], t)) for t, r in enumerate(c["rnode"])]
    unsched = {names[i] for i in range(n) if c["unsched"][i]}
    not_ready = {names[i] for i in range(n) if not c["ready"][i]}
    lab = {names[i]: int(c["lre"][i]) for i in range(n) if c["lre"][i] >= 0}
    idx = {nm: i for i, nm in enumerate(names)}
    out = []
    for x in range(len(exe[0])):
        w = rr.reschedule_executor(names, labels, sort_zone, alloc, over, resv, unsched, not_ready, lab,
                                   (int(exe[0][x]), int(exe[1][x]), int(exe[2][x])), min_frag,
                                   {names[h] for h in host[x]} if host else set(), None if keep is None else "z%d" % keep)
        out.append(idx[w] if w is not None else -1)
    return out


@pytest.mark.parametrize("seed", [21, 22, 23])
@pytest.mark.parametrize("min_frag", [False, True])
def test_literal_chain_with_scopes(packer, seed, min_frag):
    c = literal_case(seed)
    rng = np.random.default_rng(seed)
    exe, host = executors(rng, 24, len(c["names"]))
    for keep in (None, 0, 1, 2, 7):                           # 7: a zone no node has -- every node filtered out
        got, _ = one_call(packer, c, exe, min_frag, host, keep=keep, tz=c["tz"])
        want = literal_decisions(c, exe, min_frag, host, keep)
        assert list(got) == want, (seed, keep)
        if keep is not None and keep < 3:
            assert all(c["tz"][w] == keep for w in got if w >= 0)
        if keep == 7:
            assert (got == -1).all()


def test_missing_label_refused_like_filter_nodes_to_zone(packer, gangpack):
    c = literal_case(31, missing=0.05)
    c["tz"][5] = -1
    exe, host = executors(np.random.default_rng(1), 4, len(c["names"]))
    other = int(c["tz"][6]) if c["tz"][6] >= 0 else 0
    with pytest.raises(gangpack.native.GangpackError) as ei:
        one_call(packer, c, exe, False, host, keep=other, tz=c["tz"])
    assert ei.value.status == 1 and "filterNodesToZone" in str(ei.value)
    with pytest.raises(rr.ReferenceError):
        literal_decisions(c, exe, False, host, other)
    got, _ = one_call(packer, c, exe, False, host, keep=None, tz=c["tz"])    # no scope: labels are not read
    assert list(got) == literal_decisions(c, exe, False, host, None)


def test_refusals(packer, gangpack):
    Err = gangpack.native.GangpackError
    c = make_case(41, 50, 2)
    exe, host = executors(np.random.default_rng(2), 3, 50)
    with pytest.raises(Err) as ei:
        one_call(packer, c, (np.array([-1, 0, 0]), exe[1], exe[2]), False, None)
    assert ei.value.status == 1 and "negative" in str(ei.value)
    with pytest.raises(Err) as ei:
        one_call(packer, c, (np.array([1 << 61, 0, 0]), exe[1], exe[2]), False, None)
    assert ei.value.status == 6
    with pytest.raises(Err) as ei:
        one_call(packer, c, exe, True, [[0], [50], []])
    assert ei.value.status == 1 and "host_nodes" in str(ei.value)
    with pytest.raises(Err) as ei:
        one_call(packer, c, exe, False, None, keep=0, tz=None)
    assert ei.value.status == 1 and "topology_zone" in str(ei.value)
    with pytest.raises(Err) as ei:
        one_call(packer, c, exe, False, None, keep=-2, tz=c["zid"])
    assert ei.value.status == 1
    bad = dict(c, zid=c["zid"] + 5)
    with pytest.raises(Err) as ei:
        one_call(packer, bad, exe, False, None)
    assert ei.value.status == 1 and "zone_id" in str(ei.value)
    got, amb = one_call(packer, c, (np.zeros(0, np.int64),) * 3, False, None)
    assert len(got) == 0 and len(amb) == 0


def test_no_executor_candidate(packer, recipe):
    c = make_case(51, 500, 3)
    c["unsched"] = np.ones(500, np.uint8)
    exe, host = executors(np.random.default_rng(3), 16, 500)
    for mf in (False, True):
        got, amb = one_call(packer, c, exe, mf, host)
        assert (got == -1).all() and not amb.any()


def test_context_state_untouched(packer, recipe, gangpack):
    """A resident driver snapshot and an az-aware layout behave as if the call never happened."""
    c = make_case(61, 3000, 4)
    rng = np.random.default_rng(61)
    apps = random_apps(rng, 200)
    apps["group"] = np.zeros(200, np.int32)
    exe, host = executors(rng, 32, 3000)
    # the interleaved executor Predicates run on ANOTHER cluster (more nodes, other allocatable, reservations and zones), so
    # any scratch they shared with held state would be overwritten with different bytes
    o = make_case(62, 5000, 7, R=30000)
    oexe, ohost = executors(rng, 32, 5000)
    # gp_prepare_cluster + FIFO + gp_reserve_placements(subtract), then an interleaved executor Predicate
    for p, interleave in ((packer, True), (recipe, False)):
        p.prepare_cluster(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c))
        placed = p.pack_batch(apps, 0, 1)
        p.reserve_placements(apps, placed)
        if interleave:
            for mf in (False, True):
                one_call(p, o, oexe, mf, ohost)
    for x, y in zip(packer.get_snapshot(), recipe.get_snapshot()):
        assert np.array_equal(x, y)
    a, b = packer.pack_batch(apps, 0, 2), recipe.pack_batch(apps, 0, 2)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for x, y in zip(packer.get_snapshot(), recipe.get_snapshot()):
        assert np.array_equal(x, y)
    # gp_prepare_cluster_zones(GP_LAYOUT_AZ_AWARE), then orders = NULL
    for p, interleave in ((packer, True), (recipe, False)):
        p.prepare_cluster_zones(c["alloc"], c["over"], c["rnode"], c["res"], *sort_args(c), layout=False)
        if interleave:
            one_call(p, o, oexe, True, ohost, keep=1, tz=o["zid"])
            one_call(p, o, oexe, False, ohost)
    a, b = packer.pack_batch_az_aware(apps), recipe.pack_batch_az_aware(apps)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    a, b = packer.pack_fifo_az_aware(apps, 1), recipe.pack_fifo_az_aware(apps, 1)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for x, y in zip(packer.get_snapshot(), recipe.get_snapshot()):
        assert np.array_equal(x, y)


def test_50k_nodes_100k_rows(packer, recipe):
    c = make_case(71, 50000, 16, R=100000)
    exe, host = executors(np.random.default_rng(71), 200, 50000)
    for mf in (False, True):
        got, _ = one_call(packer, c, exe, mf, host)
        want, _, _ = five_calls(recipe, c, exe, mf, host)
        assert np.array_equal(got, want), mf
        got1, _ = one_call(packer, c, tuple(e[:1] for e in exe), mf, host[:1])      # one executor over 50 000 nodes
        assert got1[0] == want[0]


def test_no_sort_kernel_and_one_synchronise(packer):
    import torch
    from torch.profiler import ProfilerActivity, profile
    c = make_case(81, 20000, 8, R=40000)
    exe, host = executors(np.random.default_rng(81), 64, 20000)
    one_call(packer, c, exe, False, host)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        one_call(packer, c, exe, False, host)
        one_call(packer, c, exe, True, host)
        torch.cuda.synchronize()
    kernels = {e.name for e in prof.events() if e.device_type.name == "CUDA" and "gp_" in e.name}
    assert kernels, "no kernel seen by the profiler"
    for bad in ("gp_sort_tiles", "gp_rank_by_search", "gp_split_candidates", "gp_label_keys", "gp_label_scatter", "gp_scatter_order",
                "gp_make_keys"):
        assert not any(bad in k for k in kernels), (bad, kernels)
    for want in ("gp_rp_nodes", "gp_rp_decide", "gp_usage_scatter", "gp_availability"):
        assert any(want in k for k in kernels), (want, kernels)
    syncs = [e for e in prof.events() if e.name == "cudaStreamSynchronize"]
    assert len(syncs) == 2, len(syncs)                        # one per call
