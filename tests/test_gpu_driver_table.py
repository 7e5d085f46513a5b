"""The resident driver table (gp_driver_table_reset / _update) and its two FIFO entries (gp_pack_fifo_driver_table,
gp_pack_fifo_zones_groups_driver_table).

Each call must give, bit for bit, what the per-call entry gives on the gp_apps the host builds from the same pods -- the
queue decoded from drivers.DriverMirror through filter_to_earliest_and_sort, stable in slot order, with shouldSkipDriverFifo
-- on the same prepared snapshot: queue_slot, offsets, undefined ties, driver node, ExecutorNodes of every placed driver,
zone and average efficiency (zone form), status, statistics and the snapshot left behind.  Every refusal is checked once,
with the table (the next call's identity) and the snapshot unchanged afterwards."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import drivers, native
from oracle.pyref import filter_to_earliest_and_sort

pytestmark = pytest.mark.gpu

INVALID, CAPACITY, UNREPRESENTABLE = 1, 5, 6
SEC = 10 ** 9
STATS = ("nodes_scanned", "drivers_tried", "scan_path_apps", "scan_path_nodes")
GROUPS = [f"g{i}" for i in range(4)]


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def outcome(fn):
    try:
        return 0, fn()
    except native.GangpackError as e:
        return e.status, None


def resources(rng, big_count=None):
    gpu = rng.random() < 0.2
    return {"drv": [int(rng.integers(1, 4)) * 500, int(rng.integers(1, 4)) << 30, int(gpu)],
            "exe": [int(rng.integers(1, 5)) * 500, int(rng.integers(1, 5)) << 30, int(gpu and rng.random() < 0.5)],
            "min": int(rng.integers(0, 6)) if big_count is None else big_count}


class Pods:
    """A seeded stream of pending-driver events over a DriverTable: adds, updates, deletes, unparseable annotations"""

    def __init__(self, seed, n_slots=4, groups=GROUPS, schedulers=("s0", "s1")):
        self.rng = np.random.default_rng(seed)
        self.table = drivers.DriverTable(n_slots=n_slots, n_groups=1, n_schedulers=1)
        self.groups, self.schedulers = list(groups), list(schedulers)
        self.next_uid = 0
        self.now = 1_000 * SEC

    def add(self, k=1, **kw):
        for _ in range(k):
            uid = f"d{self.next_uid}"
            self.next_uid += 1
            self.set(uid, **kw)
        return uid

    def set(self, uid, creation=None, scheduler=None, group="?", res=None, exact=True):
        r = self.rng
        if creation is None:
            creation = int(r.integers(900, 1_000)) * SEC          # whole seconds: equal creation times are common
        if scheduler is None:
            scheduler = self.schedulers[0] if r.random() < 0.85 else self.schedulers[1]
        if group == "?":
            group = self.groups[r.integers(len(self.groups))] if r.random() < 0.9 else None
        self.table.set_driver(uid, creation, scheduler, group, res if res is not None else resources(r), exact)

    def churn(self, k):
        r = self.rng
        for _ in range(k):
            live = list(self.table.rows)
            op = r.random()
            if op < 0.55 or len(live) < 4:
                self.add()
            elif op < 0.75:
                self.table.delete_driver(live[r.integers(len(live))])
            elif op < 0.8:
                self.table.set_driver(live[r.integers(len(live))], 0, "s0", None, None)    # annotations no longer parse
            else:
                self.set(live[r.integers(len(live))])

    def ages(self):
        return self.table.group_ages(30 * SEC, {"g1": 120 * SEC, "g2": -5 * SEC})


def snapshot(rng, n_nodes, n_groups):
    """a gp_set_snapshot over n_nodes nodes in n_groups instance groups, each node a driver and an executor candidate"""
    cpu = rng.integers(2, 9, n_nodes) * 1000
    mem = rng.integers(4, 17, n_nodes).astype(np.int64) << 30
    gpu = rng.integers(0, 2, n_nodes)
    grp = rng.integers(0, n_groups, n_nodes)
    order = np.argsort(grp, kind="stable").astype(np.int32)
    off = np.zeros(n_groups + 1, np.int32)
    np.cumsum(np.bincount(grp, minlength=n_groups), out=off[1:])
    return (cpu, mem, gpu, order, order, off, off)


def oracle_order(mirror, requesting_slot):
    """the Predicate form's queue by the string-level oracle: filter_to_earliest_and_sort over the mirror's rows, listed in slot
    order, then the requesting driver"""
    pods = [dict(uid=int(s), created=int(mirror.creation[s]), scheduler=int(mirror.scheduler[s]),
                 group=None if mirror.group[s] < 0 else int(mirror.group[s])) for s in np.flatnonzero(mirror.present)]
    me = next(p for p in pods if p["uid"] == requesting_slot)
    return [p["uid"] for p in filter_to_earliest_and_sort(me, pods)] + [requesting_slot]


def per_call(p, mirror, q, algo, mode):
    """today's recipe: the host-built gp_apps and gp_pack_batch"""
    slots, apps, ties, inexact = mirror.queue(**{k: v for k, v in q.items() if k != "n_slots"})
    if q.get("requesting_slot", -1) >= 0:
        assert slots.tolist() == oracle_order(mirror, q["requesting_slot"])
    if inexact:
        return UNREPRESENTABLE, None
    st, r = outcome(lambda: p.pack_batch(apps, algo, mode))
    return st, (slots, apps, ties, r)


def check_pack(p, world, snap, q, algo, mode):
    p.set_snapshot(*snap)
    st_t, got = outcome(lambda: p.pack_fifo_driver_table(q, algo, mode))
    stats_t = p.stats() if st_t == 0 else None
    snap_t = p.get_snapshot()
    p.set_snapshot(*snap)
    st_h, want = per_call(p, world.table.mirror, q, algo, mode)
    assert st_t == st_h, (st_t, st_h)
    if stats_t is not None and st_h == 0:
        stats_h = p.stats()
        assert [stats_t[k] for k in STATS] == [stats_h[k] for k in STATS]
    for a, b in zip(snap_t, p.get_snapshot()):
        assert np.array_equal(a, b)
    if st_t:
        return st_t, None
    slots, apps, ties, (drv, exe, off) = want
    assert np.array_equal(got["queue_slot"], slots) and np.array_equal(got["off"], off)
    assert got["undefined_ties"] == ties and got["n_queued"] == len(slots) and got["n_executors"] == off[-1]
    assert np.array_equal(got["driver_node"], drv)
    for i in np.flatnonzero(drv >= 0):
        assert np.array_equal(got["executor_nodes"][off[i]:off[i + 1]], exe[off[i]:off[i + 1]])
    return 0, got


def queue_args(world, requesting=None, scheduler="s0", snapshot_group=None, predicate_group=0, now=None):
    t = world.table
    q = dict(n_slots=t.size["n_slots"], enforce_after_ns=world.ages(), now=world.now if now is None else now)
    if requesting is not None:
        q.update(requesting_slot=t.slot_of(requesting), predicate_group=predicate_group)
    else:
        q.update(requesting_slot=-1, scheduler=max(t.scheduler_id(scheduler), 0), snapshot_group=snapshot_group)
    return q


@pytest.mark.parametrize("algo", [native.TIGHTLY_PACK, native.DISTRIBUTE_EVENLY])
@pytest.mark.parametrize("mode", [native.MODE_FIFO_REFERENCE, native.MODE_FIFO_EXACT])
def test_random_streams_match_the_per_call_batch(packer, algo, mode):
    rng = np.random.default_rng(7 + algo * 3 + mode)
    world = Pods(seed=100 + 10 * algo + mode)
    snap1 = snapshot(rng, 48, 1)
    snap4 = snapshot(rng, 64, 4)
    for step in range(12):
        world.churn(int(rng.integers(5, 40)))
        world.table.flush(packer)
        live = list(world.table.rows)
        for uid in [live[i] for i in rng.permutation(len(live))[:3]]:
            st, _ = check_pack(packer, world, snap1, queue_args(world, requesting=uid), algo, mode)
            assert st == 0
        sg = world.table.snapshot_groups({g: i for i, g in enumerate(GROUPS)})
        st, _ = check_pack(packer, world, snap4, queue_args(world, snapshot_group=sg), algo, mode)
        assert st == 0


@pytest.mark.parametrize("bp", [native.BP_SINGLE_AZ_TIGHTLY_PACK, native.BP_SINGLE_AZ_MINIMAL_FRAGMENTATION,
                                native.BP_AZ_AWARE_TIGHTLY_PACK])
@pytest.mark.parametrize("mode", [native.MODE_FIFO_REFERENCE, native.MODE_FIFO_EXACT])
def test_zone_packers_match_the_per_call_drain(packer, bp, mode):
    rng = np.random.default_rng(11 + bp * 2 + mode)
    n, G = 80, 3
    alloc = (rng.integers(2, 9, n) * 1000, rng.integers(4, 17, n).astype(np.int64) << 30, rng.integers(0, 2, n))
    ig = rng.integers(0, G, n).astype(np.int32)
    zone = rng.integers(0, 3, n).astype(np.int32)
    kind = native.LAYOUT_AZ_AWARE if bp == native.BP_AZ_AWARE_TIGHTLY_PACK else native.LAYOUT_SINGLE_AZ
    empty = (np.zeros(0, np.int64), np.zeros(0, np.int64))

    def prepare():
        packer.prepare_cluster_zones_groups(alloc, None, np.zeros(0, np.int32), empty, ig, G, zone_id=zone, n_zones=3, kind=kind,
                                            layout=False)
    world = Pods(seed=200 + bp * 2 + mode)
    for step in range(8):
        world.churn(int(rng.integers(5, 40)))
        world.table.flush(packer)
        live = list(world.table.rows)
        queries = [queue_args(world, snapshot_group=world.table.snapshot_groups({"g0": 0, "g1": 1, "g3": 2}))]
        queries += [queue_args(world, requesting=live[i], predicate_group=int(rng.integers(G))) for i in rng.permutation(len(live))[:2]]
        for q in queries:
            prepare()
            st_t, got = outcome(lambda: packer.pack_fifo_zones_groups_driver_table(q, bp, mode))
            stats_t, snap_t = packer.stats(), packer.get_snapshot()
            prepare()
            slots, apps, ties, inexact = world.table.mirror.queue(**{k: v for k, v in q.items() if k != "n_slots"})
            st_h, want = outcome(lambda: packer.pack_fifo_zones_groups(apps, bp, mode))
            assert st_t == st_h == 0
            stats_h = packer.stats()
            assert [stats_t[k] for k in STATS] == [stats_h[k] for k in STATS]
            for a, b in zip(snap_t, packer.get_snapshot()):
                assert np.array_equal(a, b)
            z, drv, exe, off, avg = want
            assert np.array_equal(got["queue_slot"], slots) and np.array_equal(got["off"], off) and got["undefined_ties"] == ties
            assert np.array_equal(got["zone"], z) and np.array_equal(got["driver_node"], drv)
            for i in np.flatnonzero(drv >= 0):
                assert np.array_equal(got["executor_nodes"][off[i]:off[i + 1]], exe[off[i]:off[i + 1]])
                assert np.array_equal(got["avg_efficiency"][i], avg[i])


def test_boundaries(packer):
    rng = np.random.default_rng(3)
    snap = snapshot(rng, 32, 1)
    world = Pods(seed=3)
    algo, mode = native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE
    # an empty table: the drain selects nothing
    world.table.flush(packer)
    st, got = check_pack(packer, world, snap, queue_args(world, snapshot_group=np.zeros(1, np.int32)), algo, mode)
    assert st == 0 and got["n_queued"] == 0
    # a requesting driver without an instance group queues alone
    world.set("lonely", creation=999 * SEC, group=None)
    world.add(5, group="g0")
    world.table.flush(packer)
    st, got = check_pack(packer, world, snap, queue_args(world, requesting="lonely"), algo, mode)
    assert st == 0 and list(got["queue_slot"]) == [world.table.slot_of("lonely")]
    # creation + age == now is not young; one nanosecond later it is; a negative age (g2)
    world.set("edge", creation=world.now - 30 * SEC, group="g0")
    world.set("young", creation=world.now - 30 * SEC + 1, group="g0")
    world.set("neg", creation=world.now + 4 * SEC, group="g2")
    world.set("req0", creation=world.now + 100 * SEC, group="g0")
    world.set("req2", creation=world.now + 100 * SEC, group="g2")
    world.table.flush(packer)
    for req in ("req0", "req2"):
        st, got = check_pack(packer, world, snap, queue_args(world, requesting=req), algo, mode)
        assert st == 0
    slots, apps, _, _ = world.table.mirror.queue(**{k: v for k, v in queue_args(world, requesting="req0").items() if k != "n_slots"})
    young = dict(zip(slots.tolist(), apps["young"].tolist()))
    assert young[world.table.slot_of("edge")] == 0 and young[world.table.slot_of("young")] == 1
    # every queued driver young, and a blocked queue: a driver no node can hold blocks the requesting one (-2)
    big = {"drv": [10 ** 9, 1 << 50, 0], "exe": [1, 1, 0], "min": 1}
    for now, want in ((0, -1), (world.now + 10 ** 4 * SEC, -2)):
        w2 = Pods(seed=5)
        w2.set("blocker", creation=10 * SEC, group="g0", res=big)
        w2.set("me", creation=20 * SEC, group="g0", res=big)
        w2.table.flush(packer)
        st, got = check_pack(packer, w2, snap, queue_args(w2, requesting="me", now=now), algo, mode)
        assert st == 0 and got["driver_node"][-1] == want
    # counts at the FIFO limit 2^20 and one above it
    for k, want_st in ((1 << 20, 0), ((1 << 20) + 1, UNREPRESENTABLE)):
        w3 = Pods(seed=6)
        w3.set("many", creation=10 * SEC, group="g0", res={"drv": [1, 1, 0], "exe": [1, 1, 0], "min": k})
        w3.table.flush(packer)
        st, _ = check_pack(packer, w3, snap, queue_args(w3, requesting="many"), algo, mode)
        assert st == want_st


def test_refusals_leave_table_and_snapshot(packer):
    rng = np.random.default_rng(9)
    snap = snapshot(rng, 32, 1)
    world = Pods(seed=9)
    world.add(20, group="g0", scheduler="s0")
    world.table.flush(packer)
    t = world.table
    req = list(t.rows)[-1]
    q = queue_args(world, requesting=req)
    packer.set_snapshot(*snap)
    before = packer.pack_fifo_driver_table(q, native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE)
    base = t.delta()
    assert len(base["slot"]) == 0
    S = t.size["n_slots"]

    def one_row(**over):
        d = {k: (v[:0] if isinstance(v, np.ndarray) else v) for k, v in base.items()}
        row = dict(slot=0, present=1, creation=1, scheduler=0, group=0, drv_cpu_milli=1, drv_mem_bytes=1, drv_gpu=0, exe_cpu_milli=1,
                   exe_mem_bytes=1, exe_gpu=0, min_executor_count=1, exact=1)
        row.update(over)
        for k, v in row.items():
            d[k] = np.array([v], d[k].dtype)
        return d
    bad = [(one_row(slot=S), INVALID), (one_row(group=t.size["n_groups"]), INVALID), (one_row(group=-2), INVALID),
           (one_row(scheduler=t.size["n_schedulers"]), INVALID), (one_row(drv_mem_bytes=1 << 61), UNREPRESENTABLE)]
    dup = one_row()
    for k in dup:
        if isinstance(dup[k], np.ndarray):
            dup[k] = np.concatenate([dup[k], dup[k]])
    bad.append((dup, INVALID))
    for d, want in bad:
        st, _ = outcome(lambda: packer.driver_table_update(d))
        assert st == want
    # the refused deltas left the table as it was
    packer.set_snapshot(*snap)
    again = packer.pack_fifo_driver_table(q, native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE)
    for k in ("queue_slot", "off", "driver_node"):
        assert np.array_equal(again[k], before[k])
    # a present row with 2^62 marked inexact is accepted; a queue that selects it is refused before the pack
    world.set("huge", creation=1 * SEC, group="g0", scheduler="s0", res={"drv": [1 << 62, 1, 0], "exe": [1, 1, 0], "min": 1}, exact=False)
    t.flush(packer)
    packer.set_snapshot(*snap)
    snap_before = packer.get_snapshot()
    st, _ = outcome(lambda: packer.pack_fifo_driver_table(q, native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE))
    assert st == UNREPRESENTABLE
    for a, b in zip(snap_before, packer.get_snapshot()):
        assert np.array_equal(a, b)
    t.delete_driver("huge")
    t.flush(packer)
    # an absent requesting slot
    free = t.size["n_slots"] - 1
    assert t._uid_at.get(free) is None
    st, _ = outcome(lambda: packer.pack_fifo_driver_table(dict(q, requesting_slot=free), native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE))
    assert st == INVALID
    # both capacity refusals write the sizes needed; the retry then succeeds
    for caps in ((2, None), (None, 1)):
        st, _ = outcome(lambda: packer.pack_fifo_driver_table(q, native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE, queue_cap=caps[0],
                                                              exec_cap=caps[1], retry=False))
        assert st == CAPACITY
        for a, b in zip(snap_before, packer.get_snapshot()):
            assert np.array_equal(a, b)
        packer.set_snapshot(*snap)
        got = packer.pack_fifo_driver_table(q, native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE, queue_cap=caps[0], exec_cap=caps[1])
        for k in ("queue_slot", "off", "driver_node"):
            assert np.array_equal(got[k], before[k])
        packer.set_snapshot(*snap)


def test_replay_after_overflow_keeps_results(packer):
    rng = np.random.default_rng(12)
    snap = snapshot(rng, 32, 1)
    world = Pods(seed=12, n_slots=1)
    for _ in range(5):
        world.churn(30)
        world.table.flush(packer)
        live = list(world.table.rows)
        st, _ = check_pack(packer, world, snap, queue_args(world, requesting=live[-1]), native.DISTRIBUTE_EVENLY,
                           native.MODE_FIFO_EXACT)
        assert st == 0
    assert world.table.replays > 1


def test_config4_size_drain(packer):
    """BASELINE config 4's shape: 10 000 nodes, 50 000 pending drivers in 16 instance groups, drained in one call"""
    rng = np.random.default_rng(4)
    G = 16
    snap = snapshot(rng, 10_000, G)
    names = [f"ig{i}" for i in range(G)]
    world = Pods(seed=4, n_slots=1 << 16, groups=names, schedulers=("s0",))
    for i in range(50_000):
        world.set(f"d{i}", creation=int(rng.integers(0, 3600)) * SEC, scheduler="s0", group=names[i % G])
    world.table.flush(packer)
    sg = world.table.snapshot_groups({g: i for i, g in enumerate(names)})
    st, got = check_pack(packer, world, snap, queue_args(world, snapshot_group=sg), native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE)
    assert st == 0 and got["n_queued"] == 50_000 and got["undefined_ties"] > 0


def test_empty_drain_leaves_stats_as_the_per_call_entry(packer):
    """a drain that selects nothing returns before any pack work, as gp_pack_batch and gp_pack_fifo_zones_groups do for
    n_apps = 0: the statistics and error word of the last pack stay as they were"""
    rng = np.random.default_rng(21)
    snap = snapshot(rng, 32, 1)
    world = Pods(seed=21)
    world.add(12, group="g0", scheduler="s0")
    world.table.flush(packer)
    none = world.table.snapshot_groups({})                  # no group drained
    packer.set_snapshot(*snap)
    packer.pack_fifo_driver_table(queue_args(world, requesting=list(world.table.rows)[-1]), native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE)
    before = packer.stats()
    got = packer.pack_fifo_driver_table(queue_args(world, snapshot_group=none), native.TIGHTLY_PACK, native.MODE_FIFO_REFERENCE)
    assert got["n_queued"] == 0
    after_table = packer.stats()
    packer.pack_batch({k: np.zeros(0, np.int64) for k in drivers.QUANTITIES} | {"count": np.zeros(0, np.int32)}, native.TIGHTLY_PACK,
                      native.MODE_FIFO_REFERENCE)
    after_host = packer.stats()
    assert [after_table[k] for k in STATS] == [before[k] for k in STATS] == [after_host[k] for k in STATS]
