"""The host side of the resident reservation table, without a device: random ResourceReservation and soft-store event streams
(creates, updates, compaction rewrites, deletes, nodes leaving the cluster, capacities that grow from 1 and force replays)
through reservations.ReservationTable's deltas into the numpy ReservationMirror.  After every step the mirror's per-call
encoding (to_usage_rows), summed per node, equals the string-keyed restatement of GetReservedResources."""
import numpy as np
import pytest

from k8s_spark_scheduler_b200 import reservations as rv


class Driver:
    """A ReservationTable and the mirror its deltas build"""

    def __init__(self, n_slots=1, n_node_ids=1):
        self.table = rv.ReservationTable(n_slots=n_slots, n_node_ids=n_node_ids)
        self.mirror = rv.ReservationMirror()
        self.replays = 0

    def step(self):
        d = self.table.delta()
        self.replays += d["reset"] is not None
        self.mirror.apply(d)
        return d


def quantity(rng, big=False):
    if big:
        return int(rng.integers(-(1 << 58), 1 << 58))
    return int(rng.integers(-3, 1000)) if rng.random() < 0.1 else int(rng.integers(0, 64_000))


def entries(rng, nodes, prefix, k, big=False):
    return {f"{prefix}-{j}": (nodes[rng.integers(len(nodes))], quantity(rng, big), quantity(rng, big) << (0 if big else 10), int(rng.integers(0, 3)))
            for j in range(k)}


def churn(rng, drv, all_nodes, steps, per_step, big=False):
    """Random events, per_step of them between deltas; yields each delta after it is mirrored"""
    t = drv.table
    for s in range(steps):
        for _ in range(per_step):
            x = rng.random()
            if x < 0.35:                                        # a new or rewritten ResourceReservation
                key = ("ns", f"app-{rng.integers(12)}")
                t.rr_set(key, entries(rng, all_nodes, f"{key[1]}-e", int(rng.integers(1, 6)), big))
            elif x < 0.45 and t.rrs:                            # the compaction rewrite: same entries, some values changed
                key = list(t.rrs)[rng.integers(len(t.rrs))]
                cur = dict(t.rrs[key])
                name = list(cur)[rng.integers(len(cur))]
                node, cpu, mem, gpu = cur[name]
                cur[name] = (node, cpu + 1, mem, gpu)
                t.rr_set(key, cur)
            elif x < 0.6 and t.rrs:
                t.rr_delete(list(t.rrs)[rng.integers(len(t.rrs))])
            elif x < 0.85:                                      # soft reservations of an application: added or removed pods
                app = f"app-{rng.integers(12)}"
                cur = dict(t.soft.get(app, {}))
                if cur and rng.random() < 0.4:
                    del cur[list(cur)[rng.integers(len(cur))]]
                cur.update(entries(rng, all_nodes, f"{app}-s{s}", int(rng.integers(0, 3)), big))
                t.soft_set(app, cur)
            elif t.soft:
                t.soft_delete(list(t.soft)[rng.integers(len(t.soft))])
        yield drv.step()


def sums_per_node(mirror, nodes, node_ids):
    res_node, vals = rv.to_usage_rows(mirror, node_ids)
    out = {n: [0, 0, 0] for n in nodes}
    for r, i in enumerate(res_node.tolist()):
        if i >= 0:
            for k in range(3):
                out[nodes[i]][k] += int(vals[k][r])
    return out


def restated(table, nodes):
    usage = rv.reserved_resources(table.rrs, table.soft)
    return {n: usage.get(n, [0, 0, 0]) for n in nodes}


@pytest.mark.parametrize("seed", range(12))
def test_random_streams_match_restatement(seed):
    rng = np.random.default_rng(seed)
    all_nodes = [f"n{i}" for i in range(2 + seed % 7)]
    drv = Driver()
    for _ in churn(rng, drv, all_nodes, steps=40, per_step=1 + seed % 5):
        present = [n for n in all_nodes if rng.random() < 0.8]          # nodes that left the cluster keep their rows
        rng.shuffle(present)
        ids = drv.table.node_ids(present)
        assert sums_per_node(drv.mirror, present, ids) == restated(drv.table, present)
    assert drv.replays >= 3                                             # capacities grew from 1


def test_lost_delta_is_replayed():
    rng = np.random.default_rng(5)
    nodes = ["a", "b", "c"]
    drv = Driver(n_slots=64, n_node_ids=64)
    list(churn(rng, drv, nodes, steps=5, per_step=4))
    drv.table.rr_set(("ns", "lost"), {"x": ("a", 7, 7, 0)})
    drv.table.delta()                                                   # never applied
    drv.table.replay()
    d = drv.step()
    assert d["reset"] is not None
    assert sums_per_node(drv.mirror, nodes, drv.table.node_ids(nodes)) == restated(drv.table, nodes)


def test_slots_and_node_ids_are_reused():
    t = rv.ReservationTable(n_slots=4, n_node_ids=2)
    t.rr_set(("ns", "a"), {"d": ("n1", 1, 1, 0), "e": ("n2", 1, 1, 0)})
    t.delta()
    t.rr_delete(("ns", "a"))
    t.soft_set("b", {"p": ("n3", 2, 2, 0), "q": ("n3", 2, 2, 0)})
    d = t.delta()
    assert d["reset"] is None and t.size == dict(n_slots=4, n_node_ids=2)
    assert sorted(d["slot"].tolist()) == [0, 1] and set(d["node_id"].tolist()) == {t.node_ids(["n3"])[0]}
    assert t.node_ids(["n1", "n2"]).tolist() == [-1, -1]


def test_unchanged_entries_send_nothing():
    t = rv.ReservationTable()
    t.rr_set(("ns", "a"), {"d": ("n1", 1, 2, 3)})
    t.delta()
    t.rr_set(("ns", "a"), {"d": ("n1", 1, 2, 3)})
    t.soft_delete("absent")
    assert len(t.delta()["slot"]) == 0


def test_large_values_sum_exactly():
    rng = np.random.default_rng(11)
    nodes = ["n0", "n1"]
    drv = Driver()
    for _ in churn(rng, drv, nodes, steps=10, per_step=6, big=True):
        assert sums_per_node(drv.mirror, nodes, drv.table.node_ids(nodes)) == restated(drv.table, nodes)
