"""The host side of the resident reservation table (gp_reservation_table_*): GetReservedResources' rows kept as the shim's
ResourceReservation-cache and soft-store handlers see them, and turned into the deltas of gp_reservation_table_update.

GetReservedResources (EXT/resourcereservations.go:258-263) sums every ResourceReservation's Spec.Reservations entry
(UsageForNodes, LIB/resources/resources.go:31-43) and every soft reservation (UsedSoftReservationResources,
internal/cache/softreservations.go:155-170) per node.  Each such entry is one slot of the table here: (node id, cpu, mem, gpu).
"""
from __future__ import annotations

import numpy as np

from .overhead import _CountedInterner
from .resident import ResidentTable

_FREE = (-1, 0, 0, 0)          # node id, cpu, mem, gpu of a free slot


class ReservationTable(ResidentTable):
    """Events: rr_set((namespace, appID), {name: (node, cpu, mem, gpu)}) for a create, an update and the compaction rewrite
    alike, rr_delete(key), soft_set(appID, {pod: (node, cpu, mem, gpu)}) and soft_delete(appID).  Each entry holds one slot;
    freed slots are reused, and node ids come from a reference-counted interner, so the id of a node no entry names any more
    goes to the next new node.  delta() -> the arrays of one gp_reservation_table_update: what changed since the last delta
    (every occupied slot after a reset); see ResidentTable.  |value| >= 2^61 is refused when it arrives."""

    name, writes = "reservation", ("slot",)

    def __init__(self, n_slots=64, n_node_ids=64):
        super().__init__(ReservationMirror(), n_slots=n_slots, n_node_ids=n_node_ids)
        self.rrs, self.soft = {}, {}                    # key -> {name: (node, cpu, mem, gpu)}, as the events gave them
        self._nodes = _CountedInterner()
        self._slot = {}                                 # (kind, key, name) -> slot
        self._row, self._node = [], []                  # per slot: (node id, cpu, mem, gpu), the node name it holds (or None)
        self._free = []
        self._dirty = {}                                # slot -> the row the device holds since the last delta

    # ---- events
    def rr_set(self, key, reservations: dict):
        self._set(0, key, reservations, self.rrs)

    def rr_delete(self, key):
        self._set(0, key, {}, self.rrs)

    def soft_set(self, app, reservations: dict):
        self._set(1, app, reservations, self.soft)

    def soft_delete(self, app):
        self._set(1, app, {}, self.soft)

    # ---- queries
    def node_ids(self, nodes) -> np.ndarray:
        """the table's ids of these node names; -1 for a node no reservation names (nothing is reserved on it)"""
        return np.array([self._nodes.ids.get(n, -1) for n in nodes], np.int32)

    # ---- internals
    def _bounds(self):
        return dict(n_slots=len(self._row), n_node_ids=self._nodes.bound)

    def _changes(self, replay):
        if replay:
            slots = [at for at, row in enumerate(self._row) if row != _FREE]
        else:
            slots = sorted(at for at, was in self._dirty.items() if self._row[at] != was)
        rows = [self._row[at] for at in slots]
        d = {"slot": np.array(slots, np.int32)}
        for j, name in enumerate(("node_id", "cpu_milli", "mem_bytes", "gpu")):
            d[name] = np.array([r[j] for r in rows], np.int32 if j == 0 else np.int64)
        self._dirty = {}
        return d

    def _set(self, kind, key, reservations, store):
        old = store.pop(key, {})
        if reservations:
            store[key] = {n: tuple(r) for n, r in reservations.items()}
        for name in old.keys() - reservations.keys():
            self._write(self._slot.pop((kind, key, name)), None)
        for name, r in reservations.items():
            at = self._slot.get((kind, key, name))
            if at is None:
                at = self._free.pop() if self._free else self._grow()
                self._slot[(kind, key, name)] = at
            elif old.get(name) == tuple(r):
                continue
            self._write(at, tuple(r))

    def _grow(self):
        self._row.append(_FREE)
        self._node.append(None)
        return len(self._row) - 1

    def _write(self, at, r):
        """slot at := reservation r = (node, cpu, mem, gpu), or free it (r None)"""
        self._dirty.setdefault(at, self._row[at])
        if r is not None:
            node_id = self._nodes.acquire(r[0])         # before the release: an unchanged node keeps its id
        if self._node[at] is not None:
            self._nodes.release(self._node[at])
        if r is None:
            self._row[at], self._node[at] = _FREE, None
            self._free.append(at)
        else:
            self._row[at], self._node[at] = (node_id, int(r[1]), int(r[2]), int(r[3])), r[0]


class ReservationMirror:
    """What gp_reservation_table_update leaves on the device, with numpy: apply(delta) as the library would."""

    def __init__(self):
        self.size = None

    def apply(self, d: dict):
        if d.get("reset"):
            self.size = dict(d["reset"])
            n = self.size["n_slots"]
            self.node_id = np.full(n, -1, np.int32)
            self.v = np.zeros((3, n), np.int64)
        s = np.asarray(d["slot"], np.int64)
        ids = np.asarray(d["node_id"], np.int32)
        self.node_id[s] = ids
        for k, name in enumerate(("cpu_milli", "mem_bytes", "gpu")):
            col = d.get(name)
            self.v[k, s] = np.where(ids != -1, np.asarray(col, np.int64), 0) if col is not None else 0


def to_usage_rows(mirror: ReservationMirror, node_ids):
    """The per-call encoding of the table for a node table whose entry i carries reservation-table id node_ids[i] (-1 = none):
    one row per occupied slot, res_node = the index i with node_ids[i] == the slot's id, or -1 when no entry has it.
    -> (res_node, (cpu, mem, gpu)) as gp_usage_input takes them."""
    node_ids = np.asarray(node_ids, np.int64)
    where = np.full(mirror.size["n_node_ids"], -1, np.int32)
    known = node_ids >= 0
    where[node_ids[known]] = np.nonzero(known)[0]
    occupied = np.nonzero(mirror.node_id != -1)[0]
    res_node = where[mirror.node_id[occupied]]
    return res_node.astype(np.int32), tuple(mirror.v[k, occupied].copy() for k in range(3))


def reserved_resources(rrs: dict, soft: dict) -> dict:
    """GetReservedResources keyed by node name: node -> [cpu, mem, gpu] summed over every ResourceReservation entry
    (UsageForNodes) and every soft reservation (UsedSoftReservationResources), as Python integers."""
    usage = {}
    for entries in list(rrs.values()) + list(soft.values()):
        for node, cpu, mem, gpu in entries.values():
            u = usage.setdefault(node, [0, 0, 0])
            u[0] += cpu
            u[1] += mem
            u[2] += gpu
    return usage
