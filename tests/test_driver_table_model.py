"""drivers.DriverTable and drivers.DriverMirror against the string-level filterToEarliestAndSort
(oracle/pyref.filter_to_earliest_and_sort) over seeded pod event streams: equal timestamps, drivers without an instance
group, other schedulers, slot reuse after deletes, unparseable annotations, and the reset-and-replay that follows a
capacity overflow or a refused update."""
import numpy as np

from k8s_spark_scheduler_b200 import drivers
from oracle.pyref import filter_to_earliest_and_sort, spark_resources

SEC = 10 ** 9
GROUPS = ["a", "b", "c", "d", "e"]
SCHEDULERS = ["spark-scheduler", "other", "third"]


class FakePacker:
    """applies nothing; refuses the update after `refuse_next` is set, like a device refusal"""

    def __init__(self):
        self.resets, self.updates, self.refuse_next = [], 0, False

    def driver_table_reset(self, **size):
        self.resets.append(size)

    def driver_table_update(self, d):
        from k8s_spark_scheduler_b200.native import GangpackError
        if self.refuse_next:
            self.refuse_next = False
            raise GangpackError(1, "refused")
        self.updates += 1


def annotations(rng):
    a = {"spark-driver-cpu": str(int(rng.integers(1, 4))), "spark-driver-mem": f"{int(rng.integers(1, 8))}Gi",
         "spark-executor-cpu": str(int(rng.integers(1, 4))), "spark-executor-mem": f"{int(rng.integers(1, 8))}Gi"}
    if rng.random() < 0.3:
        a.update({"spark-dynamic-allocation-enabled": "true", "spark-dynamic-allocation-min-executor-count": str(int(rng.integers(0, 4))),
                  "spark-dynamic-allocation-max-executor-count": "9"})
    else:
        a["spark-executor-count"] = str(int(rng.integers(0, 6)))
    if rng.random() < 0.2:
        a["spark-executor-nvidia.com/gpu"] = "1"
    if rng.random() < 0.05:
        a["spark-driver-cpu"] = "not-a-quantity"
    return a


class World:
    def __init__(self, seed, n_slots=2):
        self.rng = np.random.default_rng(seed)
        self.table = drivers.DriverTable(n_slots=n_slots, n_groups=1, n_schedulers=1)
        self.packer = FakePacker()
        self.pods = {}                          # uid -> string-level pod (pyref shape) + parsed resources
        self.n = 0

    def event(self):
        r = self.rng
        live = list(self.pods)
        op = r.random()
        if op < 0.5 or not live:
            uid = f"p{self.n}"
            self.n += 1
        else:
            uid = live[r.integers(len(live))]
        if op > 0.8 and live:
            # bound, deleted or terminating: no longer a pending driver
            self.pods.pop(uid, None)
            self.table.delete_driver(uid)
            return
        err, res = spark_resources(annotations(r))
        pod = dict(uid=uid, created=int(r.integers(0, 50)) * SEC, scheduler=SCHEDULERS[r.integers(len(SCHEDULERS))],
                   group=GROUPS[r.integers(len(GROUPS))] if r.random() < 0.85 else None, node=None)
        if err:
            self.pods.pop(uid, None)           # a driver whose annotations do not parse holds no row (resource.go:232-237)
            self.table.set_driver(uid, pod["created"], pod["scheduler"], pod["group"], None)
            return
        pod["res"] = res
        self.pods[uid] = pod
        self.table.set_driver(uid, pod["created"], pod["scheduler"], pod["group"], res, res["exact"])

    def by_slot(self):
        return sorted(self.pods.values(), key=lambda p: self.table.slot_of(p["uid"]))


def uids(world, slots):
    at = {world.table.slot_of(u): u for u in world.pods}
    return [at[int(s)] for s in slots]


def check(world, now, ages):
    t, m = world.table, world.table.mirror
    age_of = {g: ages.get(g, 30 * SEC) for g in GROUPS}
    ages_arr = t.group_ages(30 * SEC, ages)
    assert set(int(s) for s in np.flatnonzero(m.present)) == {t.slot_of(u) for u in world.pods}
    for uid in list(world.pods)[:6]:
        me = world.pods[uid]
        slots, apps, ties, inexact = m.queue(requesting_slot=t.slot_of(uid), enforce_after_ns=ages_arr, now=now)
        want = filter_to_earliest_and_sort(me, world.by_slot())
        assert uids(world, slots) == [p["uid"] for p in want] + [uid]
        want_skip = [int(p["created"] + age_of[p["group"]] > now) for p in want] + [0]
        assert apps["young"].tolist() == want_skip
        for j, p in enumerate(want + [me]):
            assert [int(apps[k][j]) for k in drivers.QUANTITIES] == p["res"]["drv"] + p["res"]["exe"]
            assert int(apps["count"][j]) == p["res"]["min"]
        assert ties == sum(want[j]["created"] == want[j - 1]["created"] for j in range(1, len(want)))
    # drain form: one scheduler, groups a, c, d in snapshot groups 1, 0, 2
    index = {"a": 1, "c": 0, "d": 2}
    sched = "spark-scheduler"
    slots, apps, ties, _ = m.queue(requesting_slot=-1, scheduler=t.scheduler_id(sched), snapshot_group=t.snapshot_groups(index),
                                   enforce_after_ns=ages_arr, now=now)
    want = sorted([p for p in world.by_slot() if p["scheduler"] == sched and p["group"] in index],
                  key=lambda p: (index[p["group"]], p["created"]))
    assert uids(world, slots) == [p["uid"] for p in want]
    assert apps["group"].tolist() == [index[p["group"]] for p in want]


def test_driver_table_matches_string_level_queue():
    for seed in range(6):
        world = World(seed)
        ages = {"b": 5 * SEC, "c": -3 * SEC}
        for step in range(25):
            for _ in range(int(world.rng.integers(1, 30))):
                world.event()
            if world.rng.random() < 0.1:
                world.packer.refuse_next = True      # a refused update: the table is reset and replayed
            world.table.flush(world.packer)
            check(world, now=int(world.rng.integers(0, 60)) * SEC, ages=ages)
        assert world.table.replays > 1 and world.packer.resets


def test_slot_reuse_and_minimal_deltas():
    t = drivers.DriverTable(n_slots=8, n_groups=2, n_schedulers=1)
    res = {"drv": [1, 2, 0], "exe": [3, 4, 0], "min": 2}
    for i in range(5):
        t.set_driver(f"u{i}", i * SEC, "s", "g", res)
    assert [t.slot_of(f"u{i}") for i in range(5)] == list(range(5))
    d = t.delta()
    assert d["reset"] is not None and len(d["slot"]) == 5
    t.delete_driver("u1")
    t.delete_driver("u3")
    t.set_driver("v", 9 * SEC, "s", None, res)
    assert t.slot_of("v") == 1                      # the lowest freed slot
    t.set_driver("u0", 0, "s", "g", res)            # unchanged: not resent
    d = t.delta()
    assert d["reset"] is None and d["slot"].tolist() == [1, 3]
    assert d["present"].tolist() == [1, 0] and d["group"].tolist()[0] == -1
    t.set_driver("w", 1, "s", "g", res)
    t.delete_driver("w")                            # added and deleted before a flush: nothing to send
    assert len(t.delta()["slot"]) == 0


def test_overflow_doubles_and_replays():
    t = drivers.DriverTable(n_slots=1, n_groups=1, n_schedulers=1)
    res = {"drv": [1, 1, 0], "exe": [1, 1, 0], "min": 0}
    for i in range(9):
        t.set_driver(f"u{i}", i, f"s{i % 3}", f"g{i % 5}", res)
    d = t.delta()
    assert d["reset"] == {"n_slots": 16, "n_groups": 8, "n_schedulers": 4}
    assert sorted(d["slot"].tolist()) == list(range(9))
    t.mirror.apply(d)
    assert t.mirror.present.sum() == 9 and t.mirror.group.tolist()[:5] == [0, 1, 2, 3, 4]
