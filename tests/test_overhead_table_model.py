"""CPU checks of the resident overhead table's host side: overhead.OverheadTable turns pod, lister, ResourceReservation and
soft-store events into deltas, overhead.TableMirror applies them as the device would, and after every delta
evaluate(to_encoding(mirror)) must equal evaluate(encode(views)) -- per node name, has_reservation per slot and n_warned --
and both must equal the string restatement (tests/overhead_ref.py) fed the same pod events."""
import numpy as np
import pytest

import overhead_ref as ref
from k8s_spark_scheduler_b200 import overhead as oh
from test_overhead_model import _random_cluster, pod

SPARK = "spark-scheduler"


class Driver:
    """One OverheadTable, its mirror and the restatement, fed the same events"""

    def __init__(self, **size):
        self.table = oh.OverheadTable(**size) if size else oh.OverheadTable()
        self.mirror = oh.TableMirror()
        self.comp = ref.OverheadComputer()
        self.replays = 0

    def pod_event(self, kind, *args):
        getattr(self.table, kind)(*args)
        getattr(self.comp, "on_" + kind)(*args)

    def step(self):
        """-> the delta, applied to the mirror"""
        d = self.table.delta()
        self.replays += d["reset"] is not None
        self.mirror.apply(d)
        return d

    def expected(self, nodes):
        t = self.table
        ov, ns, warned = self.comp.get_overhead_by_node(nodes, t.lister, t.rrs, t.soft)
        return ref.columns(nodes, ov), ref.columns(nodes, ns), warned

    def check(self, nodes, query=None):
        """after a step: the table's answer (through `query`, the mirror by default) == encode(views) == the restatement"""
        t = self.table
        want_ov, want_ns, want_has, want_warned = oh.evaluate(oh.encode(t.slots, t.lister, t.rrs, t.soft, nodes))
        query = query or (lambda ids: oh.evaluate(oh.to_encoding(self.mirror, ids)))
        ov, ns, has, warned = t.answer(nodes, query)
        assert lists(ov) == lists(want_ov) and lists(ns) == lists(want_ns)
        assert warned == want_warned
        n = len(t.slots)
        assert np.array_equal(has[:n], want_has) and not has[n:].any()
        r_ov, r_ns, r_warned = self.expected(nodes)
        assert (lists(ov), lists(ns), warned) == (tuple(r_ov), tuple(r_ns), r_warned)
        return ov, ns, has, warned


def lists(triple):
    return tuple(list(map(int, c)) for c in triple)


def churn(rng, drv, n_nodes, steps, per_step, nss=("ns0", "ns1", "ns2"), apps=6, names=60):
    """Random events with churn: pods added bound or unbound, bound, unbound, updated and deleted (slots reused); lister
    entries appearing, vanishing and changing labels, role and scheduler; RRs created, rewritten with repeated names and
    deleted; soft entries set and removed; appIDs shared across namespaces.  Yields after every delta."""
    live, uid = {}, 0                                            # uid -> the pod's current object

    def make(ns=None):
        labels = {}
        if rng.random() < 0.8:
            labels["spark-app-id"] = f"app{rng.integers(apps)}"
        if rng.random() < 0.7:
            labels["spark-role"] = "executor" if rng.random() < 0.7 else "driver"
        init = [tuple(int(x) for x in rng.integers(0, 2000, 3))] if rng.random() < 0.3 else ()
        return pod(ns or nss[rng.integers(len(nss))], f"p{rng.integers(names)}", f"n{rng.integers(n_nodes + 2)}",
                   int(rng.integers(0, 4000)), int(rng.integers(0, 1 << 34)), int(rng.integers(0, 3)), labels,
                   SPARK if rng.random() < 0.6 else "other", init)

    all_names = lambda: [f"p{i}" for i in range(names)] + ["zz"]
    for _ in range(steps):
        for _ in range(per_step):
            op = rng.integers(12)
            t = drv.table
            if op <= 2 or not live:                              # a new pod, bound or not
                p = make()
                p["uid"] = f"u{uid}"
                uid += 1
                if rng.random() < 0.25:
                    p["nodeName"] = ""
                drv.pod_event("add", p)
                live[p["uid"]] = p
                if rng.random() < 0.8:
                    t.lister_set(p)
            elif op == 3:                                        # bind an unbound pod, or update a bound one
                p = live[list(live)[rng.integers(len(live))]]
                q = dict(p, nodeName=p["nodeName"] or f"n{rng.integers(n_nodes + 2)}")
                if p["nodeName"]:
                    q["containers"] = [{"cpu": 999, "memory": 99}]
                drv.pod_event("update", p, q)
                live[p["uid"]] = q
            elif op == 4:                                        # unbind
                p = live[list(live)[rng.integers(len(live))]]
                q = dict(p, nodeName="")
                drv.pod_event("update", p, q)
                live[p["uid"]] = q
            elif op == 5:                                        # delete
                p = live.pop(list(live)[rng.integers(len(live))])
                drv.pod_event("delete", p)
                if rng.random() < 0.7:
                    t.lister_delete(p["namespace"], p["name"])
            elif op == 6:                                        # the lister's pod changes labels, role or scheduler
                p = live[list(live)[rng.integers(len(live))]]
                q = make(p["namespace"])
                q.update(name=p["name"], uid=p["uid"], nodeName=p["nodeName"])
                t.lister_set(q)
            elif op == 7:                                        # a lister entry vanishes
                p = live[list(live)[rng.integers(len(live))]]
                t.lister_delete(p["namespace"], p["name"])
            elif op == 8:                                        # an RR created or rewritten, names may repeat
                key = (nss[rng.integers(len(nss))], f"app{rng.integers(apps)}")
                t.rr_set(key, list(rng.choice(all_names(), int(rng.integers(0, 10)))))
            elif op == 9 and t.rrs:
                t.rr_delete(list(t.rrs)[rng.integers(len(t.rrs))])
            elif op == 10:
                t.soft_set(f"app{rng.integers(apps)}", list(rng.choice(all_names(), int(rng.integers(0, 8)))))
            elif op == 11 and t.soft:
                t.soft_delete(list(t.soft)[rng.integers(len(t.soft))])
        yield drv.step()


@pytest.mark.parametrize("seed", range(12))
def test_random_churn_streams(seed):
    rng = np.random.default_rng(seed)
    n_nodes = 1 + seed % 5
    drv = Driver(n_slots=4, n_node_ids=2, n_app_keys=2, n_app_ids=2, n_names=4)
    nodes = [f"n{i}" for i in range(n_nodes)]
    for _ in churn(rng, drv, n_nodes, steps=25, per_step=1 + seed % 6):
        drv.check(nodes)
    assert drv.replays >= 2                                       # the capacities were doubled and the state replayed


@pytest.mark.parametrize("seed", range(8))
def test_random_cluster_streams(seed):
    """_random_cluster's pods, lister, RRs and soft store arriving as events, a delta after every few"""
    rng = np.random.default_rng(500 + seed)
    pods, lister, rrs, soft, nodes, events = _random_cluster(rng, 1 + seed % 7, 5 + 9 * seed)
    drv = Driver()
    feed = [("pod",) + tuple(e) for e in events] + [("lister", p) for p in lister.values()]
    feed += [("rr", k, v) for k, v in rrs.items()] + [("soft", k, v) for k, v in soft.items()]
    order = rng.permutation(len(feed))
    for j, i in enumerate(order):
        kind, *args = feed[i]
        if kind == "pod":
            drv.pod_event(*args)
        elif kind == "lister":
            drv.table.lister_set(*args)
        elif kind == "rr":
            drv.table.rr_set(*args)
        else:
            drv.table.soft_set(*args)
        if j % 3 == 2 or j == len(order) - 1:
            drv.step()
            drv.check(nodes)
    assert drv.table.lister == lister and drv.table.rrs == rrs and drv.table.soft == soft


def test_synthetic_cluster_with_churn():
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(3, 60, 3000, big_apps=2, big_executors=200)
    drv = Driver()
    for p in pods:
        drv.pod_event("add", p)
    for p in lister.values():
        drv.table.lister_set(p)
    for k, v in rrs.items():
        drv.table.rr_set(k, v)
    for k, v in soft.items():
        drv.table.soft_set(k, v)
    first = drv.step()
    assert first["reset"] is not None and drv.table.slots == rec.slots       # PodRecords' slot numbering
    drv.check(nodes)
    rng = np.random.default_rng(1)
    for step in range(6):                                         # 1 % of the records rewritten per step
        for i in rng.choice(len(pods), len(pods) // 100, replace=False):
            p = pods[i]
            drv.pod_event("delete", p)
            q = dict(p, uid=p["uid"] + f"-r{step}", nodeName=nodes[rng.integers(len(nodes))])
            drv.pod_event("add", q)
            pods[i] = q
            if rng.random() < 0.5:
                drv.table.lister_delete(p["namespace"], p["name"])
            else:
                drv.table.lister_set(q)
        key = (f"ns-{step}", f"new-app-{step}")
        drv.table.rr_set(key, [f"new-app-{step}-exec-{e}" for e in range(20)] * 2)
        d = drv.step()
        assert d["reset"] is None and 0 < len(d["slot"]) <= 2 * (len(pods) // 100)
        assert len(d["member_kind"]) == 20 and len(d["rr_app_key"]) == 1   # one new RR: 20 distinct names, one flag
        drv.check(nodes)


def test_delta_carries_only_changes():
    drv = Driver()
    a = pod("a", "app1-exec-1", "n1", 100, 10, labels={"spark-app-id": "app1", "spark-role": "executor"}, sched=SPARK)
    drv.pod_event("add", a)
    drv.table.lister_set(a)
    drv.table.rr_set(("a", "app1"), ["app1-exec-1", "app1-exec-1", "x"])
    d = drv.step()
    assert len(d["slot"]) == 1 and d["rr_exists"].tolist() == [1] and d["member_present"].tolist() == [1, 1]
    drv.check(["n1", "n2"])
    assert drv.table.delta()["slot"].size == 0                    # nothing changed: an empty delta
    drv.table.rr_set(("a", "app1"), ["x", "app1-exec-1"])          # the same set of names: no member change
    drv.table.lister_set(dict(a))                                  # the same pod again: the same row
    d = drv.step()
    assert (len(d["slot"]), len(d["rr_app_key"]), len(d["member_kind"])) == (0, 0, 0)
    drv.table.rr_delete(("a", "app1"))
    d = drv.step()
    assert d["rr_exists"].tolist() == [0] and d["member_present"].tolist() == [0, 0]
    ov, _, _, warned = drv.check(["n1", "n2"])
    assert lists(ov) == ([100, 0], [10, 0], [0, 0]) and warned == 0


def test_ids_of_departed_names_are_reused():
    drv = Driver()
    for k in range(4):
        p = pod("a", f"old-{k}", "n1", 1, 1, labels={"spark-app-id": f"app-{k}"}, uid=f"o{k}")
        drv.pod_event("add", p)
        drv.table.lister_set(p)
    drv.step()
    bounds = (drv.table._names.bound, drv.table._apps.bound, drv.table._keys.bound)
    for k in range(4):
        p = pod("a", f"old-{k}", "n1", uid=f"o{k}")
        drv.pod_event("delete", p)
        drv.table.lister_delete("a", f"old-{k}")
        q = pod("b", f"new-{k}", "n1", 2, 2, labels={"spark-app-id": f"other-{k}"}, uid=f"n{k}")
        drv.pod_event("add", q)
        drv.table.lister_set(q)
    drv.step()
    assert (drv.table._names.bound, drv.table._apps.bound, drv.table._keys.bound) == bounds
    assert len(drv.table.slots) == 4                               # the freed slots were reused
    drv.check(["n1"])


def test_nodes_without_an_id_answer_zero():
    drv = Driver()
    p = pod("a", "p", "n1", 5, 6)
    drv.pod_event("add", p)
    drv.table.lister_set(p)
    drv.step()
    assert drv.table.node_ids(["n9", "n1"]).tolist() == [-1, 0]
    ov, ns, _, _ = drv.check(["n9", "n1", "n8"])
    assert lists(ov) == ([0, 5, 0], [0, 6, 0], [0, 0, 0])


def test_replay_after_an_update_that_did_not_go_through():
    """A delta the device never applied (refused or failed) is lost unless replay() is called: the next delta then resets
    and resends the whole state"""
    drv = Driver()
    p = pod("a", "p", "n1", 5, 6)
    drv.pod_event("add", p)
    drv.table.lister_set(p)
    drv.step()
    q = pod("a", "q", "n1", 7, 8, uid="q")
    drv.pod_event("add", q)
    drv.table.lister_set(q)
    lost = drv.table.delta()                                      # not applied to the mirror
    assert lost["reset"] is None and len(lost["slot"]) == 1
    drv.table.replay()
    d = drv.step()
    assert d["reset"] is not None and len(d["slot"]) == 2
    ov, _, _, _ = drv.check(["n1"])
    assert lists(ov) == ([12], [14], [0])


def test_zero_capacities_grow():
    drv = Driver(n_slots=0, n_node_ids=0, n_app_keys=0, n_app_ids=0, n_names=0)
    p = pod("a", "p", "n1", 5, 6, labels={"spark-app-id": "x"})
    drv.pod_event("add", p)
    drv.table.lister_set(p)
    drv.table.soft_set("x", ["p"])
    d = drv.step()
    assert d["reset"] == dict(n_slots=1, n_node_ids=1, n_app_keys=1, n_app_ids=1, n_names=1)
    drv.check(["n1"])
