"""affinity.LabelTable without a GPU: random node add / relabel / delete streams turned into label-table deltas, applied to
the numpy mirror (through flush() with a recording packer that can refuse an update), then the mirror decoded into the
per-call labels and evaluated with the table's encoding of the affinities -- which must equal the string-level Match of
tests/affinity_ref.py on every node.  Covers capacity doubling with replay, a refused update followed by a replay, id reuse
after deletes, strings no node carries, and values at and past the int64 limits."""
import numpy as np
import pytest

import affinity_ref as ar
from k8s_spark_scheduler_b200 import affinity as aff
from k8s_spark_scheduler_b200.native import GangpackError
from test_affinity_model import KEYS, VALUES, random_cluster

LIMITS = ["9223372036854775807", "-9223372036854775808", "9223372036854775808", "-9223372036854775809"]
EXTRA_KEYS = [f"others/k{i}" for i in range(12)]


class RecordingPacker:
    """label_table_reset / _update as the library takes them, kept as a list of calls; refuse_next makes the next update raise
    GP_ERR_INVALID (the library leaves the table as it was)"""

    def __init__(self):
        self.calls, self.refuse_next = [], False

    def label_table_reset(self, **size):
        self.calls.append(("reset", size))

    def label_table_update(self, d):
        if self.refuse_next:
            self.refuse_next = False
            raise GangpackError(1, "gp_label_table_update: refused")
        self.calls.append(("update", d))


def random_labels(rng):
    keys = rng.choice(KEYS[:-1] + EXTRA_KEYS, int(rng.integers(0, 14)), replace=False)
    return {str(k): str(rng.choice(VALUES + LIMITS + [f"v{int(rng.integers(0, 40))}"])) for k in keys}


def step(rng, t, live, serial):
    """one batch of node events: relabels (some to the same labels), adds and deletes"""
    for _ in range(int(rng.integers(1, 12))):
        r = rng.random()
        if r < 0.25 or not live:
            name = f"node-{serial[0]}"
            serial[0] += 1
            live.append(name)
            t.set_node(name, random_labels(rng))
        elif r < 0.4:
            name = live.pop(int(rng.integers(0, len(live))))
            t.delete_node(name)
        elif r < 0.5:
            name = live[int(rng.integers(0, len(live)))]
            t.set_node(name, dict(t.labels[name]))            # an informer update with the same labels: no write
        else:
            name = live[int(rng.integers(0, len(live)))]
            t.set_node(name, random_labels(rng))


def check(t, rng, live, n_aff=24):
    names = list(rng.permutation(live)) + ["never-seen"]
    _, affs = random_cluster(rng, 1, n_aff)
    affs.append({"nodeSelector": {"ghost-key": "a"}, "required": None})
    affs.append({"required": [{"matchExpressions": [("zone", "In", ["ghost-value", "also-ghost", "a"])]}]})
    affs.append({"required": [{"matchExpressions": [("ghost-key", "DoesNotExist", [])]}, ]})
    affs.append({"required": [{"matchExpressions": [("zone", "NotIn", ["ghost-value"])]}]})
    affs.append({"required": [{"matchExpressions": [("gpus", "Gt", ["5"])], "matchFields": [("metadata.name", "In", [names[0]])]}]})
    enc = dict(t.to_node_labels(t.node_ids(names)), **t.encode_affinities(affs, names))
    outcome = aff.evaluate(enc)[0]
    nodes = [{"name": nm, "labels": t.labels.get(nm, {})} for nm in names]
    want = np.array([[ar.outcome(p, nd) for nd in nodes] for p in affs], np.int8)
    assert np.array_equal(outcome, want)
    # no encoding of an affinity changes the table
    assert t.delta()["row_node"].size == 0 and t.delta()["value_id"].size == 0


@pytest.mark.parametrize("seed", range(8))
def test_event_streams_match_string_oracle(seed):
    rng = np.random.default_rng(seed)
    t = aff.LabelTable(n_node_ids=2, max_labels=1, n_keys=2, n_values=2)
    p = RecordingPacker()
    live, serial = [], [0]
    resets = 0
    for s in range(14):
        step(rng, t, live, serial)
        p.refuse_next = s % 5 == 3
        t.flush(p)
        resets += sum(1 for c in p.calls if c[0] == "reset")
        p.calls = []
        check(t, rng, live)
    assert resets >= 3                                        # the first, capacity doublings and the refusals' replays
    assert t.mirror.size["max_labels"] >= 8 and t.mirror.size["n_node_ids"] >= 16


def test_flush_writes_only_changed_rows_and_new_values():
    t = aff.LabelTable()
    p = RecordingPacker()
    t.set_node("a", {"zone": "x", "n": "7"})
    t.set_node("b", {"zone": "y"})
    t.flush(p)
    assert [c[0] for c in p.calls] == ["reset", "update"]
    p.calls = []
    t.set_node("a", {"n": "7", "zone": "x"})                 # same labels
    t.flush(p)
    assert p.calls == []                                       # nothing changed: no update
    t.set_node("b", {"zone": "x"})
    t.delete_node("a")
    t.set_node("c", {"zone": "z"})                            # takes a's id
    t.flush(p)
    (kind, d), = p.calls
    assert kind == "update" and d["reset"] is None
    assert sorted(d["row_node"].tolist()) == [0, 1]
    assert d["value_id"].tolist() == [t._vals["z"]]
    assert t.node_ids(["c", "b", "a"]).tolist() == [0, 1, -1]
    lab = t.to_node_labels(t.node_ids(["a", "b", "c"]))
    assert lab["label_off"].tolist() == [0, 0, 1, 2]


def test_int64_limits_parse_per_value():
    t = aff.LabelTable()
    for i, v in enumerate(LIMITS):
        t.set_node(f"n{i}", {"v": v})
    t.flush(RecordingPacker())
    lab = t.to_node_labels(t.node_ids([f"n{i}" for i in range(4)]))
    assert lab["label_int_ok"].tolist() == [1, 1, 0, 0]
    assert lab["label_int"].tolist() == [2 ** 63 - 1, -2 ** 63, 0, 0]


def test_second_refusal_is_raised():
    class Refusing(RecordingPacker):
        def label_table_update(self, d):
            raise GangpackError(1, "refused")
    t = aff.LabelTable()
    t.set_node("a", {"k": "v"})
    with pytest.raises(GangpackError):
        t.flush(Refusing())
