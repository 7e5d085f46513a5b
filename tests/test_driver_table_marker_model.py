"""drivers.DriverTable's affinity column and DriverMirror.stale against a string-level restatement of
scanForUnschedulablePods' filter (EXT/unschedulablepods.go:93-166) over seeded pod event streams: other schedulers, binding,
deletion, terminating pods, executors, unparseable annotations, affinity interning and id reuse, the reset-and-replay after
a refused update, creation + timeout == now against one nanosecond less, and int64-extreme creation and timeout values."""
import numpy as np

from k8s_spark_scheduler_b200 import drivers
from oracle.pyref import spark_resources
from test_driver_table_model import FakePacker, annotations

SEC = 10 ** 9
LO, HI = -(1 << 63), (1 << 63) - 1
SCHEDULERS = ["spark-scheduler", "other"]
AFFS = [None,
        {"nodeSelector": {}, "required": None},                           # matches every node: -1 as well
        {"nodeSelector": {"a": "1", "b": "2"}, "required": None},
        {"nodeSelector": {"b": "2", "a": "1"}, "required": None},         # the same program, keys in another order
        {"nodeSelector": None, "required": [{"matchExpressions": [("zone", "In", ["z1", "z2"])]}]},
        {"nodeSelector": None, "required": [{"matchExpressions": [("zone", "In", ["z2", "z1"])]}]},
        {"nodeSelector": None, "required": []},
        {"nodeSelector": {"a": "1"}, "required": [{"matchFields": [("metadata.name", "In", ["n3"])]}]}]


def scan_for_unschedulable_pods(pods, timeout, now):
    """the stale drivers scanForUnschedulablePods checks, by uid: spark-scheduler, role driver, pending (no node), not
    terminating, annotations that parse, CreationTimestamp.Add(timeout).Before(now)"""
    return {u for u, p in pods.items()
            if p["scheduler"] == "spark-scheduler" and p["role"] == "driver" and p["node"] is None and not p["deleting"]
            and not spark_resources(p["annotations"])[0] and p["created"] + timeout < now}


class World:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.table = drivers.DriverTable(n_slots=2, n_groups=1, n_schedulers=1)
        self.packer = FakePacker()
        self.pods = {}
        self.n = 0

    def created(self):
        r = self.rng
        u = r.random()
        if u < 0.05:
            return [LO, LO + 1, HI - 1, HI][r.integers(4)]
        return int(r.integers(0, 40)) * SEC

    def write(self, uid):
        """what the pod informer's handler does with one pod: a pending, parseable driver is set, anything else deleted"""
        p = self.pods.get(uid)
        err, res = spark_resources(p["annotations"]) if p else ("gone", None)
        if p is None or err or p["role"] != "driver" or p["node"] is not None or p["deleting"]:
            self.table.delete_driver(uid)
        else:
            self.table.set_driver(uid, p["created"], p["scheduler"], None, res, res["exact"], affinity=p["affinity"])

    def event(self):
        r = self.rng
        live = list(self.pods)
        op = r.random()
        if op < 0.45 or not live:
            uid = f"p{self.n}"
            self.n += 1
            self.pods[uid] = dict(created=self.created(), scheduler=SCHEDULERS[int(r.random() < 0.2)],
                                  role="driver" if r.random() < 0.9 else "executor", node=None, deleting=False,
                                  annotations=annotations(r), affinity=AFFS[r.integers(len(AFFS))])
        else:
            uid = live[r.integers(len(live))]
            p = self.pods[uid]
            if op < 0.55:
                p["node"] = "n0"                                # bound
            elif op < 0.65:
                del self.pods[uid]                              # deleted
            elif op < 0.7:
                p["deleting"] = True                            # terminating
            elif op < 0.85:
                p["affinity"] = AFFS[r.integers(len(AFFS))]
            else:
                p["annotations"] = annotations(r)               # may no longer parse
                p["created"] = self.created()
        self.write(uid)


def check(w, timeout, now):
    t, m = w.table, w.table.mirror
    slots, apps, outside = m.stale(t.scheduler_id("spark-scheduler"), timeout, now)
    at = {t.slot_of(u): u for u in w.pods}
    got = [at[int(s)] for s in slots]
    assert set(got) == scan_for_unschedulable_pods(w.pods, timeout, now)
    assert got == sorted(got, key=lambda u: (w.pods[u]["created"], t.slot_of(u)))
    progs = t.affinity_programs()
    for j, u in enumerate(got):
        p = w.pods[u]
        res = spark_resources(p["annotations"])[1]
        assert [int(apps[k][j]) for k in drivers.QUANTITIES] == res["drv"] + res["exe"]
        assert int(apps["count"][j]) == res["min"]
        g = int(apps["group"][j])
        key = drivers.affinity_key(p["affinity"])
        assert (g == -1) == (key is None) and (g == -1 or drivers.affinity_key(progs[g]) == key)
        assert bool(outside[j]) == (not res["exact"] or min(res["drv"] + res["exe"]) < 0 or res["min"] < 0)
    # every live id is held by some row and no two ids hold the same program
    keys = [drivers.affinity_key(a) for a in progs]
    live = set(int(a) for a in m.affinity[m.present] if a >= 0)
    assert len({k for i, k in enumerate(keys) if i in live}) == len(live)


def test_stale_matches_the_string_level_scan():
    for seed in range(6):
        w = World(seed)
        for step in range(25):
            for _ in range(int(w.rng.integers(1, 30))):
                w.event()
            if w.rng.random() < 0.1:
                w.packer.refuse_next = True                     # a refused update: the table is reset and replayed
            w.table.flush(w.packer)
            for timeout, now in ((10 * SEC, int(w.rng.integers(0, 60)) * SEC), (0, HI), (1, HI), (-1, LO), (HI, HI), (LO, LO),
                                 (LO, HI), (HI, LO)):
                check(w, timeout, now)
        assert w.table.replays > 1


def test_boundary_is_strict():
    t = drivers.DriverTable()
    res = {"drv": [1, 1, 0], "exe": [1, 1, 0], "min": 1}
    t.set_driver("edge", 100, "s", None, res)
    t.set_driver("past", 99, "s", None, res)
    t.set_driver("max", HI, "s", None, res)
    t.set_driver("min", LO, "s", None, res)
    t.mirror.apply(t.delta())
    slot = lambda slots: sorted(u for u in ("edge", "past", "max", "min") if t.slot_of(u) in slots.tolist())
    assert slot(t.mirror.stale(0, 10, 110)[0]) == ["min", "past"]          # 100 + 10 == 110 is not before 110
    assert slot(t.mirror.stale(0, 1, HI)[0]) == ["edge", "min", "past"]     # HI + 1 is not below HI (no wrap)
    assert slot(t.mirror.stale(0, -1, LO)[0]) == ["min"]                    # LO - 1 is below LO (no wrap)
    assert slot(t.mirror.stale(-1, 0, HI)[0]) == []                         # scheduler -1 selects nothing


def test_affinity_interning_counts_and_reuses_lowest_ids():
    t = drivers.DriverTable()
    res = {"drv": [1, 1, 0], "exe": [1, 1, 0], "min": 1}
    a, b, c = ({"nodeSelector": {"k": v}, "required": None} for v in "abc")
    t.set_driver("u0", 0, "s", None, res, affinity=a)
    t.set_driver("u1", 0, "s", None, res, affinity=b)
    t.set_driver("u2", 0, "s", None, res, affinity=dict(b))               # the same program: the same id
    t.set_driver("u3", 0, "s", None, res, affinity={"nodeSelector": None, "required": None})
    d = t.delta()
    assert d["affinity"].tolist() == [0, 1, 1, -1]
    t.delete_driver("u0")                                                  # id 0 freed
    t.set_driver("u1", 0, "s", None, res, affinity=None)                   # id 1 still held by u2
    t.set_driver("u4", 0, "s", None, res, affinity=c)                      # the lowest free id
    assert t.affinity_programs() == [c, b]
    d = t.delta()
    # u4 took u0's slot and id: the same record, so only u1 is sent (an id's program is given per sweep)
    assert t.slot_of("u4") == 0 and dict(zip(d["slot"].tolist(), d["affinity"].tolist())) == {1: -1}
    t.delete_driver("u2")
    t.set_driver("u5", 0, "s", None, res, affinity=a)                      # 1 is free again
    assert t.affinity_programs()[1] == a
    t.set_driver("u4", 0, "s", None, res, affinity=c)                      # unchanged: nothing sent, counts kept
    t.delta()
    assert len(t.delta()["slot"]) == 0 and t.affinity_programs() == [c, a]
