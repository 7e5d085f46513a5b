"""nodes.NodeTable against the node names themselves (no GPU): the mirror's name_rank is the byte order of the present names
after every delta, the deltas are minimal, and a new name between two keys with no gap left relabels every node."""
import random

import numpy as np
import pytest

from k8s_spark_scheduler_b200 import affinity
from k8s_spark_scheduler_b200 import nodes


def _names_rank(table):
    """the dense byte-order rank of every present node, by node id"""
    present = sorted(table.nodes, key=lambda n: n.encode())
    return {table.node_ids([n])[0]: r for r, n in enumerate(present)}


def _row(mirror, at):
    return (bool(mirror.present[at]), tuple(mirror.alloc[:, at]), int(mirror.unschedulable[at]), int(mirror.ready[at]),
            int(mirror.name_key[at]))


def _stream(seed, key_bits, steps, size=8):
    rng = random.Random(seed)
    labels = affinity.LabelTable(n_node_ids=4)
    table = nodes.NodeTable(labels, n_node_ids=4, key_bits=key_bits)
    alphabet = "abcz-0.9é"
    for step in range(steps):
        for _ in range(rng.randint(1, size)):
            op = rng.random()
            live = sorted(table.nodes)
            if op < 0.55 or not live:
                name = "".join(rng.choice(alphabet) for _ in range(rng.randint(1, 6)))
                if rng.random() < 0.3 and live:          # squeeze between two neighbours
                    a = rng.choice(live)
                    name = a + rng.choice("0a")
                labels.set_node(name, {"zone": rng.choice("xy")})
                table.set_node(name, (rng.randint(0, 64000), rng.randint(0, 1 << 40), rng.randint(0, 8)), rng.random() < 0.1,
                               rng.random() < 0.9)
            elif op < 0.75:
                name = rng.choice(live)
                table.delete_node(name)
                labels.delete_node(name)
            else:
                name = rng.choice(live)
                cpu, mem, gpu, uns, rdy = table.nodes[name]
                flip = rng.randint(0, 2)
                table.set_node(name, (cpu + (flip == 0), mem, gpu), uns if flip != 1 else not uns, rdy if flip != 2 else not rdy)
        yield step, labels, table


@pytest.mark.parametrize("seed,key_bits", [(1, 62), (2, 62), (3, 8), (4, 7), (5, 10)])
def test_name_rank_is_byte_order_and_deltas_minimal(seed, key_bits):
    relabels_seen = 0
    mirror_before = None
    for step, labels, table in _stream(seed, key_bits, steps=60):
        relabels = table.relabels
        d = table.delta()
        before = None if d["reset"] else {at: _row(table.mirror, at) for at in range(table.mirror.size["n_node_ids"])}
        table.mirror.apply(d)
        m = table.mirror
        want = _names_rank(table)
        got = {int(at): int(m.name_rank[at]) for at in np.nonzero(m.present)[0]}
        assert got == want
        assert (m.name_rank[~m.present] == -1).all()
        keys = [table.name_key(n) for n in sorted(table.nodes, key=lambda s: s.encode())]
        assert keys == sorted(set(keys)) and all(0 <= k < (1 << key_bits) for k in keys)
        if d["reset"] is None and relabels == relabels_seen:
            changed = {at for at, row in before.items() if row != _row(m, at)}
            assert set(d["node_id"].tolist()) == changed
        relabels_seen = relabels
        mirror_before = m
    assert mirror_before is not None


def test_gap_exhaustion_relabels_every_node():
    labels = affinity.LabelTable()
    table = nodes.NodeTable(labels, key_bits=4)
    for n in ("a", "c"):
        labels.set_node(n, {})
        table.set_node(n, (1, 1, 0), False, True)
    table.mirror.apply(table.delta())
    names = ["b"]
    while table.relabels == 0:
        nm = names[-1] + "b"
        names.append(nm)
        labels.set_node(nm, {})
        table.set_node(nm, (1, 1, 0), False, True)
    d = table.delta()
    assert d["reset"] is None
    assert sorted(d["node_id"].tolist()) == sorted(table.node_ids(list(table.nodes)).tolist())
    table.mirror.apply(d)
    assert {int(a): int(table.mirror.name_rank[a]) for a in np.nonzero(table.mirror.present)[0]} == _names_rank(table)


def test_unchanged_node_sends_nothing_and_ids_follow_labels():
    labels = affinity.LabelTable()
    table = nodes.NodeTable(labels)
    labels.set_node("n1", {"a": "1"})
    table.set_node("n1", (1000, 2000), False, True)
    assert table.node_ids(["n1"])[0] == labels.node_ids(["n1"])[0]
    table.mirror.apply(table.delta())
    table.set_node("n1", (1000, 2000, 0), False, True)
    assert len(table.delta()["node_id"]) == 0
    with pytest.raises(KeyError):
        table.set_node("n2", (1, 1), False, True)


def test_label_columns_follow_the_reference_rules():
    labels = affinity.LabelTable()
    spec = {"n0": {nodes.ZONE_LABEL: "z1", "ig": "g1", "pri": "hi"}, "n1": {"ig": "g9", "pri": "lo"}, "n2": {nodes.ZONE_LABEL: "z0"}}
    for n, lab in spec.items():
        labels.set_node(n, lab)
    labels.mirror.apply(labels.delta())
    args = nodes.label_args(labels, zones=["z0", "z1"], instance_group_label="ig", instance_groups=["g1", "g2"],
                            driver_priority=("pri", ["hi", "lo", "hi"]), executor_priority=("absent", ["x"]))
    cols = nodes.label_columns(labels.mirror, labels.node_ids(list(spec)), **args)
    assert cols["zone_id"].tolist() == [1, 2, 0]              # n1 has no zone label: "default", appended as zone 2
    assert cols["instance_group"].tolist() == [0, -1, -1]
    assert cols["driver_label_rank"].tolist() == [2, 1, -1]    # "hi" listed twice: its last index
    assert cols["executor_label_rank"].tolist() == [-1, -1, -1]
    with pytest.raises(ValueError):
        nodes.label_columns(labels.mirror, labels.node_ids(list(spec)), **dict(args, zone_missing=-1))


def test_misuse_is_refused_without_changing_the_table():
    labels = affinity.LabelTable()
    table = nodes.NodeTable(labels, key_bits=2)          # keys 0..3
    for n in ("b", "d"):
        labels.set_node(n, {})
        table.set_node(n, (1, 1, 0), False, True)
    labels.delete_node("b")                              # the label table first: "b" comes back under another id
    labels.set_node("x", {})                             # takes b's freed id
    labels.set_node("b", {})
    with pytest.raises(ValueError):
        table.set_node("b", (2, 2, 0), False, True)
    for n in ("a", "c", "e", "f"):
        labels.set_node(n, {})
    table.delete_node("b")
    for n in ("a", "c", "e"):                            # keys 0, 1, 3 around d's 2: no gap after e
        table.set_node(n, (1, 1, 0), False, True)
    keys = dict(table._key), list(table._sorted)
    with pytest.raises(OverflowError):                   # a fifth name: a relabel would need 5 keys of 4
        table.set_node("f", (1, 1, 0), False, True)
    assert (dict(table._key), list(table._sorted)) == keys and "f" not in table.nodes
    table.mirror.apply(table.delta())
    assert {int(a): int(table.mirror.name_rank[a]) for a in np.nonzero(table.mirror.present)[0]} == _names_rank(table)
