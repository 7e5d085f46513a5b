"""nodes.NodeTable's creation column and the failover reconciler's instance-group decoding (no GPU).

Creation times round-trip through the deltas into the mirror; a changed creation time makes exactly its row dirty, an
unchanged one none; replay resends every row with its creation time.  reconcile_groups() over the label mirror equals the
reference's instanceGroup(n.Labels[instanceGroupLabel]) on the label strings: a missing label and "" are one group, a value
not listed is refused, and so is a missing label without a group for "".  Misuse is refused without changing any state."""
import random

import numpy as np
import pytest

from k8s_spark_scheduler_b200 import affinity
from k8s_spark_scheduler_b200 import nodes

IG = "instance-group"


def _world(seed, n=60):
    rng = random.Random(seed)
    labels = affinity.LabelTable(n_node_ids=4)
    table = nodes.NodeTable(labels, n_node_ids=4)
    strings = {}
    for i in range(n):
        name = f"n{rng.randint(0, 10 ** 6)}"
        lab = {}
        if rng.random() < 0.8:
            lab[IG] = rng.choice(["a", "b", "c", ""])
        strings[name] = lab
        labels.set_node(name, lab)
        table.set_node(name, (1000, 1 << 30, 0), False, True, creation=rng.choice([0, 5, 5, 7, 1 << 62]))
    return rng, labels, table, strings


def _flush(labels, table):
    labels.mirror.apply(labels.delta())
    table.mirror.apply(table.delta())


def test_creation_round_trip_dirty_rows_and_replay():
    rng, labels, table, strings = _world(1)
    _flush(labels, table)
    names = sorted(table.nodes)
    ids = table.node_ids(names)
    cols = table.mirror.to_columns(ids)
    assert list(cols["creation"]) == [table.creation[n] for n in names]
    # the same creation time again: nothing to send; a new one: exactly that row
    table.set_node(names[0], (1000, 1 << 30, 0), False, True, creation=table.creation[names[0]])
    assert len(table.delta()["node_id"]) == 0
    table.set_node(names[1], (1000, 1 << 30, 0), False, True, creation=table.creation[names[1]] + 1)
    d = table.delta()
    assert list(d["node_id"]) == [ids[1]] and list(d["creation"]) == [table.creation[names[1]]]
    table.mirror.apply(d)
    # a creation changed and changed back before a flush is not sent
    c = table.creation[names[2]]
    table.set_node(names[2], (1000, 1 << 30, 0), False, True, creation=c + 9)
    table.set_node(names[2], (1000, 1 << 30, 0), False, True, creation=c)
    assert len(table.delta()["node_id"]) == 0
    # a deleted row is written absent with creation 0; replay resends every creation time
    table.delete_node(names[3])
    d = table.delta()
    assert list(d["node_id"]) == [ids[3]] and list(d["creation"]) == [0] and list(d["present"]) == [0]
    table.mirror.apply(d)
    assert table.mirror.creation[ids[3]] == 0
    table.replay()
    d = table.delta()
    assert d["reset"] is not None
    got = dict(zip(d["node_id"].tolist(), d["creation"].tolist()))
    assert got == {int(table.node_ids([n])[0]): table.creation[n] for n in table.nodes}
    fresh = nodes.NodeMirror()
    fresh.apply(d)
    left = sorted(table.nodes)
    assert np.array_equal(fresh.to_columns(table.node_ids(left))["creation"], table.mirror.to_columns(table.node_ids(left))["creation"])


def test_delta_without_creation_reads_zero():
    m = nodes.NodeMirror()
    m.apply(dict(reset=dict(n_node_ids=2), node_id=[1], present=[1], alloc_cpu_milli=[1], alloc_mem_bytes=[1], alloc_gpu=[0],
                 unschedulable=[0], ready=[1], name_key=[3]))
    assert m.to_columns([1])["creation"].tolist() == [0]


def _reference_groups(strings, names, groups):
    """instanceGroup(n.Labels[instanceGroupLabel]) per node: the index of the string in groups ("" for a missing label)"""
    return [groups.index(strings[n].get(IG, "")) if strings[n].get(IG, "") in groups else None for n in names]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reconcile_groups_follow_the_label_strings(seed):
    rng, labels, table, strings = _world(seed)
    _flush(labels, table)
    names = sorted(table.nodes)
    ids = table.node_ids(names)
    for groups in (["a", "b", "c"], ["c", "", "b", "a"], ["b", "a", "c", "zz"]):
        args = nodes.reconcile_label_args(labels, IG, groups)
        full = groups + ([""] if "" not in groups else [])
        assert args["n_groups"] == len(full) and args["instance_group_missing"] == full.index("")
        got = nodes.reconcile_groups(labels.mirror, ids, **args)
        assert got.tolist() == _reference_groups(strings, names, full)
    # a missing label and "" are one group
    blank = [i for i, n in enumerate(names) if strings[n].get(IG) == ""]
    missing = [i for i, n in enumerate(names) if IG not in strings[n]]
    assert blank and missing
    g = nodes.reconcile_groups(labels.mirror, ids, **nodes.reconcile_label_args(labels, IG, ["a", "b", "c"]))
    assert len({int(g[i]) for i in blank + missing}) == 1
    # no instance-group label configured: every node in group 0
    assert nodes.reconcile_groups(labels.mirror, ids).tolist() == [0] * len(ids)


def test_reconcile_groups_refusals_leave_the_tables():
    rng, labels, table, strings = _world(4)
    _flush(labels, table)
    names = sorted(table.nodes)
    ids = table.node_ids(names)
    before = (table.delta(), labels.delta())
    args = nodes.reconcile_label_args(labels, IG, ["a", "b", "c"])
    with pytest.raises(ValueError):                                   # "c" is carried but not listed
        nodes.reconcile_groups(labels.mirror, ids, **dict(args, instance_group_value=args["instance_group_value"][[0, 1, 3]]))
    with pytest.raises(ValueError):                                   # a missing label without a group for ""
        nodes.reconcile_groups(labels.mirror, ids, **dict(args, instance_group_missing=-1))
    # misuse of the node table: an unknown node, or a name under a freed id
    with pytest.raises(KeyError):
        table.set_node("no-such-node", (1, 1, 0), False, True, creation=3)
    assert "no-such-node" not in table.creation
    assert len(before[0]["node_id"]) == 0 and len(table.delta()["node_id"]) == 0
    assert len(labels.delta()["row_node"]) == 0
