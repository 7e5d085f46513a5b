"""The resident driver table (gp_driver_table_* of include/gangpack.h) from the pod informer's events, and the per-call FIFO
queue a driver-table entry stands for.

DriverTable keeps, per pending driver pod, what the device's driver table holds: the creation time (UnixNano), the
scheduler and instance-group ids (the host interns Spec.SchedulerName and FindInstanceGroupFromPodSpec's group; -1 when no
group is found), the six quantities of sparkResources, MinExecutorCount, whether every quantity is exact and the id of its
required node affinity (interned by a canonical key; -1 for no nodeSelector and no required affinity).  A driver is
written only while it is pending and its annotations parse; a bound, deleted or terminating driver, and one whose
annotations no longer parse, is deleted.  Slots freed by a delete are reused, lowest first.

DriverMirror is a numpy copy of what the device holds.  queue() decodes it into the gp_apps the per-call path builds:
filterToEarliestAndSort (EXT/sparkpods.go:54-71, stable in slot order) for the Predicate form, every drained row in
(snapshot group, creation, slot) order for the drain form, and shouldSkipDriverFifo for skip_if_no_fit.  stale() decodes it
into what the unschedulable-pod marker's sweep selects (scanForUnschedulablePods, EXT/unschedulablepods.go:93-166): the
drivers of one scheduler with creation + timeout < now, in (creation, slot) order, with their gp_apps columns and which of
them lie outside the capacity check's model.
"""
from __future__ import annotations

import heapq

import numpy as np

from .resident import ResidentTable

QUANTITIES = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu")
DELTA_COLUMNS = ("drv_cpu_milli", "drv_mem_bytes", "drv_gpu", "exe_cpu_milli", "exe_mem_bytes", "exe_gpu")
_ABSENT = (False, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0, False, -1)
MATCH_ALL = {"nodeSelector": None, "required": None}


def affinity_key(affinity):
    """A canonical, hashable key of a required-affinity program in the form LabelTable.encode_affinities takes, or None for
    one that matches every node (no nodeSelector and no required terms)"""
    if affinity is None:
        return None
    sel = tuple(sorted((affinity.get("nodeSelector") or {}).items()))
    terms = affinity.get("required")
    if not sel and terms is None:
        return None
    req = None if terms is None else tuple(
        tuple(tuple((k, op, tuple(vs)) for k, op, vs in (t.get(part) or ())) for part in ("matchExpressions", "matchFields"))
        for t in terms)
    return sel, req


class DriverTable(ResidentTable):
    """Every pending driver as the resident driver table keeps it: set_driver(uid, creation, scheduler, group, resources,
    exact, affinity) for an add or an update (resources None: the annotations do not parse, so the driver is deleted),
    delete_driver(uid) when it is bound, deleted or terminating.  resources is sparkResources' dict ({"drv": [cpu, mem, gpu],
    "exe": [...], "min": MinExecutorCount}); affinity the pod's required node affinity in the form
    affinity.LabelTable.encode_affinities takes ({"nodeSelector": ..., "required": ...}), or None.  Distinct affinities are
    interned by affinity_key with reference counts, a freed id reused lowest first; affinity_programs() lists them by id.

    delta() -> the arrays of one gp_driver_table_update: the slots that changed; see ResidentTable."""

    name, writes = "driver", ("slot",)

    def __init__(self, n_slots=64, n_groups=4, n_schedulers=2):
        super().__init__(DriverMirror(), n_slots=int(n_slots), n_groups=int(n_groups), n_schedulers=int(n_schedulers))
        self.rows = {}                                  # uid -> the row as a delta writes it
        self._slot, self._uid_at = {}, {}               # uid -> slot, slot -> uid
        self._free, self._next = [], 0                  # freed slots (a heap), the first slot never used
        self.schedulers, self.groups = {}, {}           # interners: name -> id
        self._aff_id, self._aff_refs, self._aff_prog = {}, {}, {}   # affinity key -> id, id -> live rows, id -> program
        self._aff_free, self._aff_next = [], 0
        self._dirty = set()
        self._sent = {}                                 # slot -> the row the device holds

    # ---- events
    def set_driver(self, uid, creation, scheduler, group, resources, exact=True, affinity=None):
        if resources is None:
            self.delete_driver(uid)
            return
        sid = self._intern(self.schedulers, scheduler)
        gid = -1 if group is None else self._intern(self.groups, group)
        q = [int(v) for v in resources["drv"]] + [int(v) for v in resources["exe"]]
        old = self.rows.get(uid)
        aid = self._aff_acquire(affinity)
        if old is not None:
            self._aff_release(old[12])
        row = (True, int(creation), sid, gid, *q, int(resources["min"]), bool(exact), aid)
        if old == row:
            return
        if uid not in self._slot:
            s = heapq.heappop(self._free) if self._free else self._take_new()
            self._slot[uid] = s
            self._uid_at[s] = uid
        self.rows[uid] = row
        self._dirty.add(self._slot[uid])

    def delete_driver(self, uid):
        s = self._slot.pop(uid, None)
        if s is None:
            return
        self._aff_release(self.rows[uid][12])
        del self.rows[uid], self._uid_at[s]
        heapq.heappush(self._free, s)
        self._dirty.add(s)

    # ---- queries
    def slot_of(self, uid) -> int:
        """the driver's slot, -1 when the table holds no row for it"""
        return self._slot.get(uid, -1)

    def affinity_programs(self) -> list:
        """the interned affinities by id (an id no live driver holds: a program that matches every node), for
        affinity.LabelTable.encode_affinities; the gp_node_affinities of a marker sweep"""
        return [self._aff_prog.get(a, MATCH_ALL) for a in range(self._aff_next)]

    def scheduler_id(self, name) -> int:
        """the id of a scheduler name, -1 for a name no driver has carried (a drain of it selects nothing)"""
        return self.schedulers.get(name, -1)

    def group_ages(self, default_ns, overrides=None) -> np.ndarray:
        """enforce_after_ns [n_groups]: the override of each group id's name, else DefaultEnforceAfterPodAge"""
        ages = np.full(self.size["n_groups"], int(default_ns), np.int64)
        for name, g in self.groups.items():
            if overrides and name in overrides:
                ages[g] = int(overrides[name])
        return ages

    def snapshot_groups(self, group_index) -> np.ndarray:
        """snapshot_group [n_groups] of the drain form: group_index maps an instance-group name to its snapshot group; every
        other group id is -1 (not drained)"""
        sg = np.full(self.size["n_groups"], -1, np.int32)
        for name, g in self.groups.items():
            if name in group_index:
                sg[g] = int(group_index[name])
        return sg

    # ---- internals
    def _bounds(self):
        return dict(n_slots=self._next, n_groups=len(self.groups), n_schedulers=len(self.schedulers))

    def _changes(self, replay):
        if replay:
            self._sent = {}
            slots = sorted(self._uid_at)
        else:                                           # a row changed and changed back (or added and deleted) is not sent
            slots = [s for s in sorted(self._dirty) if self._record(s) != self._sent.get(s, _ABSENT)]
        rec = [self._record(s) for s in slots]
        for s, r in zip(slots, rec):
            self._sent[s] = r
        col = lambda j, dt: np.array([r[j] for r in rec], dt)
        d = {"slot": np.array(slots, np.int32), "present": col(0, np.uint8),
             "creation": col(1, np.int64), "scheduler": col(2, np.int32), "group": col(3, np.int32)}
        for j, k in enumerate(DELTA_COLUMNS):
            d[k] = col(4 + j, np.int64)
        d["min_executor_count"] = col(10, np.int32)
        d["exact"] = col(11, np.uint8)
        d["affinity"] = col(12, np.int32)
        self._dirty = set()
        return d

    def _take_new(self):
        s = self._next
        self._next += 1
        return s

    def _aff_acquire(self, affinity):
        key = affinity_key(affinity)
        if key is None:
            return -1
        a = self._aff_id.get(key)
        if a is None:
            a = heapq.heappop(self._aff_free) if self._aff_free else self._aff_next
            self._aff_next = max(self._aff_next, a + 1)
            self._aff_id[key], self._aff_prog[a], self._aff_refs[a] = a, affinity, 0
        self._aff_refs[a] += 1
        return a

    def _aff_release(self, a):
        if a < 0:
            return
        self._aff_refs[a] -= 1
        if self._aff_refs[a] == 0:
            del self._aff_refs[a], self._aff_id[affinity_key(self._aff_prog.pop(a))]
            heapq.heappush(self._aff_free, a)

    @staticmethod
    def _intern(table, name):
        if name not in table:
            table[name] = len(table)
        return table[name]

    def _record(self, s):
        uid = self._uid_at.get(s)
        return _ABSENT if uid is None else self.rows[uid]


class DriverMirror:
    """What gp_driver_table_update leaves on the device, with numpy: apply(delta) as the library would."""

    def __init__(self):
        self.size = None

    def apply(self, d: dict):
        if d.get("reset"):
            self.size = dict(d["reset"])
            S = self.size["n_slots"]
            self.present = np.zeros(S, bool)
            self.exact = np.zeros(S, bool)
            self.creation = np.zeros(S, np.int64)
            self.scheduler = np.zeros(S, np.int32)
            self.group = np.full(S, -1, np.int32)
            self.q = np.zeros((6, S), np.int64)
            self.count = np.zeros(S, np.int32)
            self.affinity = np.full(S, -1, np.int32)
        s = np.asarray(d["slot"], np.int64)
        on = np.asarray(d["present"], np.uint8) != 0
        self.present[s] = on
        self.exact[s] = on & (np.asarray(d["exact"], np.uint8) != 0)
        self.creation[s] = np.where(on, np.asarray(d["creation"], np.int64), 0)
        self.scheduler[s] = np.where(on, np.asarray(d["scheduler"], np.int32), 0)
        self.group[s] = np.where(on, np.asarray(d["group"], np.int32), -1)
        for j, k in enumerate(DELTA_COLUMNS):
            self.q[j, s] = np.where(on, np.asarray(d[k], np.int64), 0)
        self.count[s] = np.where(on, np.asarray(d["min_executor_count"], np.int32), 0)
        aff = d.get("affinity")
        self.affinity[s] = np.where(on, np.asarray(aff, np.int32), -1) if aff is not None else -1

    def queue(self, requesting_slot=-1, scheduler=0, predicate_group=0, snapshot_group=None, enforce_after_ns=None, now=0):
        """The per-call queue of one gp_driver_queue: -> (queue_slot, apps, undefined_ties, inexact), apps the gp_apps columns
        (QUANTITIES, count, group, young = skip_if_no_fit, off) in queue order, inexact = a queued row has exact = 0.
        Raises KeyError for an absent requesting slot."""
        ages = np.zeros(0, np.int64) if enforce_after_ns is None else np.asarray(enforce_after_ns, np.int64)
        live = np.flatnonzero(self.present)
        if requesting_slot >= 0:
            if not (requesting_slot < len(self.present) and self.present[requesting_slot]):
                raise KeyError(requesting_slot)
            # filterToEarliestAndSort: same scheduler, same instance group (none matches nothing), created strictly earlier;
            # a stable sort by creation over the slot order
            g = self.group[requesting_slot]
            keep = live[(self.scheduler[live] == self.scheduler[requesting_slot]) & (self.group[live] == g) & (g >= 0) &
                        (self.creation[live] < self.creation[requesting_slot])]
            earlier = keep[np.argsort(self.creation[keep], kind="stable")].tolist()
            order = earlier + [int(requesting_slot)]
            sgs = [int(predicate_group)] * len(order)
            skip = [self._young(s, ages, now) for s in order[:-1]] + [False]
        else:
            sgm = np.asarray(snapshot_group, np.int32)
            keep = live[(self.scheduler[live] == scheduler) & (self.group[live] >= 0)]
            keep = keep[sgm[self.group[keep]] >= 0]
            order = keep[np.lexsort((self.creation[keep], sgm[self.group[keep]]))].tolist()   # stable: slot order among equal keys
            sgs = sgm[self.group[np.array(order, np.int64)]].tolist() if order else []
            skip = [self._young(s, ages, now) for s in order]
        o = np.array(order, np.int64)
        apps = {k: self.q[j, o].copy() for j, k in enumerate(QUANTITIES)}
        apps["count"] = self.count[o].copy()
        apps["group"] = np.array(sgs, np.int32)
        apps["young"] = np.array(skip, np.uint8)
        apps["off"] = np.zeros(len(o) + 1, np.int64)
        np.cumsum(np.maximum(apps["count"], 0), out=apps["off"][1:])
        cre = self.creation[o]
        ties = int(np.sum((cre[1:] == cre[:-1]) & (apps["group"][1:] == apps["group"][:-1]))) if len(o) > 1 else 0
        inexact = bool(len(o) and not self.exact[o].all())
        return o.astype(np.int32), apps, ties, inexact

    def stale(self, scheduler, timeout_ns, now, n_aff=None):
        """The marker's sweep restated per call: the present rows of `scheduler` with creation + timeout_ns < now (Python
        integers: exact), in (creation, slot) order.  -> (slots, apps, outside): apps the gp_apps columns (QUANTITIES, count
        and group = the affinity id, -1 replaced by n_aff when given) of every stale row, outside = the row has exact = 0, a
        negative quantity or a negative count (what the capacity check refuses)."""
        live = np.flatnonzero(self.present & (self.scheduler == scheduler))
        keep = [int(s) for s in live if int(self.creation[s]) + int(timeout_ns) < int(now)]
        o = np.array(sorted(keep, key=lambda s: (int(self.creation[s]), s)), np.int64)
        apps = {k: self.q[j, o].copy() for j, k in enumerate(QUANTITIES)}
        apps["count"] = self.count[o].copy()
        g = self.affinity[o].copy()
        if n_aff is not None:
            g[g == -1] = n_aff
        apps["group"] = g
        outside = ~self.exact[o] | (self.q[:, o] < 0).any(axis=0) | (self.count[o] < 0)
        return o.astype(np.int32), apps, outside

    def _young(self, s, ages, now):
        """shouldSkipDriverFifo: creation + enforce-after age > now, with Python integers (exact)"""
        return int(self.creation[s]) + int(ages[self.group[s]]) > int(now)
