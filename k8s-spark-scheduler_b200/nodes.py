"""The resident node table (gp_node_table_* of include/gangpack.h) from the node informer's events, and the per-call columns
a node-table Predicate stands for.

NodeTable keeps, per node, what the device's node table holds: allocatable, Spec.Unschedulable, the NodeReady condition,
the creation time (metav1.Time as UnixNano, the failover reconciler's newest-first order) and name_key, an order key of the
node's name.  Node ids are those of an affinity.LabelTable, so one node event feeds both
tables.  name_key is strictly increasing in the byte order of the names: a new name takes the midpoint of its neighbours'
keys, and when no gap is left every present node is relabelled with evenly spaced keys in one delta.  The device recomputes
each row's dense rank from the keys, so no Predicate sorts names.

label_columns() decodes zone, instance group and the two label priority ranks from an affinity.LabelMirror with the
reference's rules (resources.go:78-81 for the zone and its "default" placeholder, nodesorting.go:161-189 for the ranks), and
label_args() builds the per-call arguments of the node-table entries from the label strings.  reconcile_groups() and
reconcile_label_args() do the same for the failover reconciler's instance groups, instanceGroup(n.Labels[label]), where a
node without the label is in the group of "".
"""
from __future__ import annotations

import bisect

import numpy as np

from .resident import ResidentTable

ZONE_LABEL = "failure-domain.beta.kubernetes.io/zone"
DEFAULT_ZONE = "default"


_ABSENT = (False, 0, 0, 0, False, False, 0, 0)


class NodeTable(ResidentTable):
    """Every node's allocatable, unschedulable and ready flags, creation time and name order, as the resident node table keeps
    them: set_node(name, allocatable, unschedulable, ready, creation) for an add or an update (after the label table's set_node, which
    gives the node its id; nothing changes when the values are the same), delete_node(name) (before the label table's
    delete_node, which frees the id).

    delta() -> the arrays of one gp_node_table_update: the rows of the nodes that changed (a deleted node's row written
    absent), or every present row after a relabel; see ResidentTable.  key_bits bounds the keys to [0, 2^key_bits); a
    smaller value makes relabels frequent (tests)."""

    name, writes = "node", ("node_id",)

    def __init__(self, labels, n_node_ids=64, key_bits=62):
        super().__init__(NodeMirror(), n_node_ids=n_node_ids)
        self.labels = labels
        self._key_hi = 1 << key_bits
        self.nodes = {}                                 # name -> (cpu, mem, gpu, unschedulable, ready)
        self.creation = {}                              # name -> creation time (UnixNano)
        self._id, self._key = {}, {}                    # name -> node id, name -> name_key
        self._name_at = {}                              # node id -> name
        self._sorted = []                               # the present names' bytes, ascending
        self._dirty = set()
        self._sent = {}                                 # node id -> the row the device holds (as _record gives it)
        self.relabels = 0

    # ---- events
    def set_node(self, name, allocatable, unschedulable, ready, creation=0):
        at = self.labels._node.get(name)
        if at is None:
            raise KeyError(f"node {name!r} has no label-table id: LabelTable.set_node first")
        if self._name_at.get(at, name) != name:
            raise ValueError(f"node id {at} is still held by {self._name_at[at]!r}: delete_node it first")
        if self._id.get(name, at) != at:
            raise ValueError(f"node {name!r} is held under node id {self._id[name]}, not the label table's {at}: delete_node it "
                             "before the label table's delete_node")
        cpu, mem = int(allocatable[0]), int(allocatable[1])
        gpu = int(allocatable[2]) if len(allocatable) > 2 and allocatable[2] is not None else 0
        row = (cpu, mem, gpu, bool(unschedulable), bool(ready))
        if self.nodes.get(name) == row and self.creation.get(name) == int(creation) and self._id.get(name) == at:
            return
        if name not in self._id:
            self._insert(name)
        self.nodes[name] = row
        self.creation[name] = int(creation)
        self._id[name] = at
        self._name_at[at] = name
        self._dirty.add(at)

    def delete_node(self, name):
        at = self._id.pop(name, None)
        if at is None:
            return
        del self.nodes[name], self.creation[name], self._name_at[at], self._key[name]
        b = name.encode()
        del self._sorted[bisect.bisect_left(self._sorted, b)]
        self._dirty.add(at)

    # ---- queries
    def node_ids(self, names) -> np.ndarray:
        """the table's ids of these node names (-1 for a node the table does not hold)"""
        return np.array([self._id.get(n, -1) for n in names], np.int32)

    def name_key(self, name) -> int:
        return self._key[name]

    # ---- internals
    def _bounds(self):
        return dict(n_node_ids=max(self._name_at, default=-1) + 1)

    def _changes(self, replay):
        if replay:
            self._sent = {}
            rows = sorted(self._name_at)
        else:                                           # a row changed and changed back (or added and deleted) is not sent
            rows = [at for at in sorted(self._dirty) if self._record(at) != self._sent.get(at, _ABSENT)]
        rec = [self._record(at) for at in rows]
        for at, r in zip(rows, rec):
            self._sent[at] = r
        d = {"node_id": np.array(rows, np.int32),
             "present": np.array([r[0] for r in rec], np.uint8), "alloc_cpu_milli": np.array([r[1] for r in rec], np.int64),
             "alloc_mem_bytes": np.array([r[2] for r in rec], np.int64), "alloc_gpu": np.array([r[3] for r in rec], np.int64),
             "unschedulable": np.array([r[4] for r in rec], np.uint8), "ready": np.array([r[5] for r in rec], np.uint8),
             "name_key": np.array([r[6] for r in rec], np.int64), "creation": np.array([r[7] for r in rec], np.int64)}
        self._dirty = set()
        return d

    def _record(self, at):
        """the row of node id `at` as a delta writes it"""
        nm = self._name_at.get(at)
        if nm is None:
            return _ABSENT
        return (True, *self.nodes[nm], self._key[nm], self.creation[nm])

    def _insert(self, name):
        # keys lie in [0, 2^key_bits): -1 and 2^key_bits stand for the neighbours past either end
        b = name.encode()
        k = bisect.bisect_left(self._sorted, b)
        lo = self._key[self._sorted[k - 1].decode()] if k > 0 else -1
        hi = self._key[self._sorted[k].decode()] if k < len(self._sorted) else self._key_hi
        if hi - lo >= 2:
            self._sorted.insert(k, b)
            self._key[name] = (lo + hi) // 2
            return
        # no gap left: evenly spaced keys for every present name, all sent in the next delta
        n = len(self._sorted) + 1
        step = self._key_hi // (n + 1)
        if step < 1:
            raise OverflowError("more nodes than name keys (key_bits too small)")
        self._sorted.insert(k, b)
        for j, s in enumerate(self._sorted):
            nm = s.decode()
            self._key[nm] = step * (j + 1)
            if nm in self._id:
                self._dirty.add(self._id[nm])
        self.relabels += 1


class NodeMirror:
    """What gp_node_table_update leaves on the device, with numpy: apply(delta) as the library would, name_rank included."""

    def __init__(self):
        self.size = None

    def apply(self, d: dict):
        if d.get("reset"):
            self.size = dict(d["reset"])
            R = self.size["n_node_ids"]
            self.present = np.zeros(R, bool)
            self.alloc = np.zeros((3, R), np.int64)
            self.unschedulable = np.zeros(R, np.uint8)
            self.ready = np.zeros(R, np.uint8)
            self.name_key = np.zeros(R, np.int64)
            self.creation = np.zeros(R, np.int64)
        ids = np.asarray(d["node_id"], np.int64)
        on = np.asarray(d["present"], np.uint8) != 0
        self.present[ids] = on
        for j, k in enumerate(("alloc_cpu_milli", "alloc_mem_bytes", "alloc_gpu")):
            self.alloc[j, ids] = np.where(on, np.asarray(d[k], np.int64), 0)
        self.unschedulable[ids] = np.where(on, np.asarray(d["unschedulable"], np.uint8) != 0, 0)
        self.ready[ids] = np.where(on, np.asarray(d["ready"], np.uint8) != 0, 0)
        self.name_key[ids] = np.where(on, np.asarray(d["name_key"], np.int64), 0)
        cre = d.get("creation")
        self.creation[ids] = np.where(on, np.asarray(cre, np.int64), 0) if cre is not None else 0
        keys = np.where(self.present, self.name_key, np.iinfo(np.int64).max)
        order = np.lexsort((np.arange(len(keys)), keys))
        self.name_rank = np.full(len(keys), -1, np.int32)
        self.name_rank[order] = np.arange(len(keys), dtype=np.int32)
        self.name_rank[~self.present] = -1

    def to_columns(self, node_table_id) -> dict:
        """the per-call columns of the listed nodes: alloc (cpu, mem, gpu), name_rank (a permutation of 0..n-1 in the order
        of the table's ranks), unschedulable, ready, creation"""
        ids = np.asarray(node_table_id, np.int64)
        if not self.present[ids].all():
            raise ValueError("a listed node is not in the node table")
        rank = np.empty(len(ids), np.int32)
        rank[np.argsort(self.name_rank[ids], kind="stable")] = np.arange(len(ids), dtype=np.int32)
        return dict(alloc=tuple(self.alloc[d, ids].copy() for d in range(3)), name_rank=rank,
                    unschedulable=self.unschedulable[ids].copy(), ready=self.ready[ids].copy(), creation=self.creation[ids].copy())


def _value_of(mirror, ids, key):
    """per listed node: the value id of label `key` in its label-table row (-1 without it, or for an id the table lacks)"""
    if key < 0:
        return np.full(len(ids), -1, np.int64)
    R = len(mirror.count)
    ok = (ids >= 0) & (ids < R)
    rows = np.where(ok, ids, 0)
    hit = (mirror.key[rows] == key) & (np.arange(mirror.key.shape[1]) < mirror.count[rows][:, None]) & ok[:, None]
    return np.where(hit.any(1), mirror.val[rows, hit.argmax(1)], -1).astype(np.int64)


def _index_of(vals, lst):
    """per value: its index in lst (the last one of a repeated value, as valueRanks[value] = i keeps), -1 for -1 or a value
    not listed"""
    pos = {int(v): i for i, v in enumerate(lst if lst is not None else [])}
    if not pos:
        return np.full(len(vals), -1, np.int32)
    k = np.array(sorted(pos), np.int64)
    v = np.array([pos[x] for x in k], np.int32)
    j = np.clip(np.searchsorted(k, vals), 0, len(k) - 1)
    return np.where((vals >= 0) & (k[j] == vals), v[j], -1).astype(np.int32)


def label_columns(mirror, node_table_id, zone_key=-1, zone_value=None, zone_missing=-1, instance_group_key=-1,
                  instance_group_value=None, driver_rank_key=-1, driver_rank_value=None, executor_rank_key=-1,
                  executor_rank_value=None, **_):
    """The columns a node-table entry reads from the label table, decoded from an affinity.LabelMirror with its rules (the
    keyword arguments of native.GangPacker's *_node_table nodes dict; others are ignored): zone_id (None with zone_key -1),
    instance_group (None with instance_group_key -1), driver_label_rank and executor_label_rank (None when not configured).
    A zone the call would refuse raises ValueError."""
    ids = np.asarray(node_table_id, np.int64)
    out = dict(zone_id=None, instance_group=None)
    if zone_key >= 0:
        v = _value_of(mirror, ids, zone_key)
        z = np.where(v < 0, zone_missing, _index_of(v, zone_value)).astype(np.int32)
        if (z < 0).any():
            raise ValueError("a zone label value not in zone_value, or a node without the zone label (zone_missing = -1)")
        out["zone_id"] = z
    if instance_group_key >= 0:
        out["instance_group"] = _index_of(_value_of(mirror, ids, instance_group_key), instance_group_value)
    for name, key, lst in (("driver_label_rank", driver_rank_key, driver_rank_value),
                           ("executor_label_rank", executor_rank_key, executor_rank_value)):
        out[name] = None if key < 0 else _index_of(_value_of(mirror, ids, key), lst)
    return out


def label_args(labels, zones=None, zone_label=ZONE_LABEL, instance_group_label=None, instance_groups=None, driver_priority=None,
               executor_priority=None) -> dict:
    """The label arguments of a node-table entry's nodes dict from the strings, against an affinity.LabelTable's interners:
    zones, the zone names in dense-id order (a node without zone_label is in "default", which is appended when not listed);
    instance_groups, the instance-group label values in instance-group order; driver_priority / executor_priority, a
    (label name, DescendingPriorityValues) pair or None.  A string no node carries gets a negative value id, which no row
    holds."""
    def key(k):
        return labels._keys.get(k, -1) if k is not None else -1

    unknown = iter(range(-1, -(1 << 30), -1))

    def vals(lst):
        return np.array([labels._vals[v] if v in labels._vals else next(unknown) for v in lst], np.int32)

    zones = list(zones or [])
    if DEFAULT_ZONE not in zones:
        zones.append(DEFAULT_ZONE)
    # key id 0 is the label table's id of a string no node carries: a configured label that no node has
    args = dict(zone_key=key(zone_label), n_zones=len(zones), zone_value=vals(zones), zone_missing=zones.index(DEFAULT_ZONE))
    if args["zone_key"] < 0:                            # no node carries the zone label: every node is in "default"
        args.update(zone_key=-1, n_zones=1, zone_value=None, zone_missing=-1)
    if instance_group_label is not None:
        args.update(instance_group_key=max(key(instance_group_label), 0), instance_group_value=vals(instance_groups or []))
    for pfx, pr in (("driver", driver_priority), ("executor", executor_priority)):
        if pr is not None:
            args.update({f"{pfx}_rank_key": max(key(pr[0]), 0), f"{pfx}_rank_value": vals(pr[1])})
    return args


def reconcile_groups(mirror, node_table_id, instance_group_key=-1, instance_group_value=None, instance_group_missing=-1, **_):
    """The failover reconciler's instance group of each listed node, as gp_reconcile_find_nodes_node_table reads it from an
    affinity.LabelMirror: the index of its instance_group_key value in instance_group_value, instance_group_missing (the
    group of "") for a node without the label, 0 for every node with instance_group_key -1.  A group the call would refuse
    (a value not listed, or a missing label with instance_group_missing -1) raises ValueError."""
    ids = np.asarray(node_table_id, np.int64)
    if instance_group_key < 0:
        return np.zeros(len(ids), np.int32)
    v = _value_of(mirror, ids, instance_group_key)
    g = np.where(v < 0, instance_group_missing, _index_of(v, instance_group_value)).astype(np.int32)
    if (g < 0).any():
        raise ValueError("an instance-group label value not in instance_group_value, or a node without the label "
                         "(instance_group_missing = -1)")
    return g


def reconcile_label_args(labels, instance_group_label, instance_groups) -> dict:
    """The instance-group arguments of reconcile_find_nodes_node_table from the strings: instance_groups, the label values
    in instance-group order; "" (the group of a node without the label) is appended when not listed.  -> dict(
    instance_group_key, instance_group_value, instance_group_missing, n_groups)."""
    groups = list(instance_groups)
    if "" not in groups:
        groups.append("")
    args = label_args(labels, instance_group_label=instance_group_label, instance_groups=groups)
    return dict(instance_group_key=args["instance_group_key"], instance_group_value=args["instance_group_value"],
                instance_group_missing=groups.index(""), n_groups=len(groups))
