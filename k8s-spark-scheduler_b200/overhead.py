"""The overhead computer (internal/extender/overhead.go) over gp_node_overhead (include/gangpack.h).

The event side stays on the host, as in the reference: PodRecords keeps one record slot per pod the pod informer added with
spec.nodeName set (addPodRequests, overhead.go:163-174, reached through the informer's nodeName filter, so the update that
binds a pod is an add), holding its namespace, name and podToResources at that event; deletePodRequests (:176-193) frees the
slot.  encode() interns the strings of the records, the pod lister's current pods, the ResourceReservations and the soft
store into the arrays of gp_node_overhead; the device does the per-call side (computeNodeOverhead, :120-153) for every
listed node at once.  evaluate() runs the encoded arrays with numpy: the reference semantics over ids, used as a check of the
device and as a host baseline.

Descriptions:
    pod         {"uid", "namespace", "name", "labels": {str: str}, "schedulerName", "nodeName",
                 "containers": [{"cpu": millicores, "memory": bytes, "nvidia.com/gpu": units}], "initContainers": [...]}
                (only these three resources count; other request keys are ignored)
    lister      {(namespace, name): pod}                      the pod lister's current pods
    rrs         {(namespace, appID): [Status.Pods values]}    the ResourceReservation cache
    soft        {appID: [Reservations keys]}                  the soft-reservation store (keyed by appID alone)
    nodes       [node name]                                   the listed nodes, in node-table order
"""
from __future__ import annotations

import numpy as np

from .resident import ResidentTable

SPARK_APP_ID_LABEL = "spark-app-id"
SPARK_ROLE_LABEL = "spark-role"
EXECUTOR = "executor"
SPARK_SCHEDULER_NAME = "spark-scheduler"
_DIMS = ("cpu", "memory", "nvidia.com/gpu")
_MAX = 1 << 61


def pod_to_resources(pod) -> tuple:
    """podToResources (overhead.go:195-209): the containers' requests summed, then a per-dimension max with each init
    container's requests (Resources.SetMaxResource)."""
    res = [0, 0, 0]
    for c in pod.get("containers", ()):
        for d, k in enumerate(_DIMS):
            res[d] += int(c.get(k, 0))
    for c in pod.get("initContainers", ()):
        for d, k in enumerate(_DIMS):
            res[d] = max(res[d], int(c.get(k, 0)))
    return tuple(res)


class PodRecords:
    """Record slots maintained from pod informer events, the way a shim keeps them for gp_node_overhead: a slot per
    (node, UID) -- the reference's ClusterRequests map -- and a free list.  slots[i] is None for a free slot."""

    def __init__(self):
        self.slots = []
        self._free = []
        self._at = {}

    def add(self, pod):
        """informer OnAdd through the nodeName filter"""
        if pod.get("nodeName"):
            self._record(pod)

    def update(self, old, new):
        """informer OnUpdate through the nodeName filter: unbound -> bound is an add, bound -> unbound a delete; an update
        of a bound pod changes nothing (the record keeps the requests of its add)"""
        if new.get("nodeName") and not old.get("nodeName"):
            self._record(new)
        elif old.get("nodeName") and not new.get("nodeName"):
            self._remove(old)

    def delete(self, pod):
        if pod.get("nodeName"):
            self._remove(pod)

    def _record(self, pod):
        key = (pod["nodeName"], pod["uid"])
        at = self._at.get(key)
        if at is None:
            if self._free:
                at = self._free.pop()
            else:
                at = len(self.slots)
                self.slots.append(None)
            self._at[key] = at
        self.slots[at] = (pod["namespace"], pod["name"], pod["nodeName"], pod_to_resources(pod))

    def _remove(self, pod):
        at = self._at.pop((pod["nodeName"], pod["uid"]), None)
        if at is not None:
            self.slots[at] = None
            self._free.append(at)


class _Interner(dict):
    def id(self, key):
        v = self.get(key)
        if v is None:
            v = self[key] = len(self)
        return v


def encode(slots, lister, rrs, soft, nodes) -> dict:
    """Intern the strings into the arrays of gp_node_overhead.  slots: PodRecords.slots (or the same tuples
    (namespace, name, nodeName, (cpu, mem, gpu)) / None).  -> dict with the gp_overhead_pods and gp_overhead_reservations
    fields, the n_* sizes and node_ids (the listed nodes)."""
    node_ix, key_ix, app_ix, name_ix = _Interner(), _Interner(), _Interner(), _Interner()
    node_ids = np.array([node_ix.id(n) for n in nodes], np.int32)
    rr_items = list(rrs.items())
    rr_app_key = np.array([key_ix.id(k) for k, _ in rr_items], np.int32)
    rr_pod_off = np.zeros(len(rr_items) + 1, np.int64)
    np.cumsum([len(v) for _, v in rr_items], out=rr_pod_off[1:])
    rr_pod_name = np.array([name_ix.id(s) for _, v in rr_items for s in v], np.int32)
    soft_items = list(soft.items())
    soft_app_id = np.array([app_ix.id(k) for k, _ in soft_items], np.int32)
    soft_pod_off = np.zeros(len(soft_items) + 1, np.int64)
    np.cumsum([len(v) for _, v in soft_items], out=soft_pod_off[1:])
    soft_pod_name = np.array([name_ix.id(s) for _, v in soft_items for s in v], np.int32)
    n = len(slots)
    node_id = np.full(n, -1, np.int32)
    req = np.zeros((3, n), np.int64)
    listed = np.zeros(n, np.uint8)
    app_key = np.full(n, -1, np.int32)
    app_id = np.full(n, -1, np.int32)
    name_id = np.zeros(n, np.int32)
    is_executor = np.zeros(n, np.uint8)
    spark = np.zeros(n, np.uint8)
    for i, rec in enumerate(slots):
        if rec is None:
            continue
        ns, name, node, r = rec
        node_id[i] = node_ix.id(node)
        req[:, i] = r
        pod = lister.get((ns, name))
        if pod is None:
            continue
        listed[i] = 1
        labels = pod.get("labels") or {}
        app = labels.get(SPARK_APP_ID_LABEL)
        if app is not None:
            app_key[i] = key_ix.id((pod["namespace"], app))
            app_id[i] = app_ix.id(app)
        name_id[i] = name_ix.id(pod["name"])
        is_executor[i] = labels.get(SPARK_ROLE_LABEL) == EXECUTOR
        spark[i] = pod.get("schedulerName") == SPARK_SCHEDULER_NAME
    return dict(n_pods=n, n_node_ids=len(node_ix), n_app_keys=len(key_ix), n_app_ids=len(app_ix), n_names=len(name_ix),
                node_id=node_id, req_cpu_milli=req[0], req_mem_bytes=req[1], req_gpu=req[2], listed=listed, app_key=app_key,
                app_id=app_id, name_id=name_id, is_executor=is_executor, spark_scheduler=spark,
                n_rr=len(rr_items), rr_app_key=rr_app_key, rr_pod_off=rr_pod_off, rr_pod_name=rr_pod_name,
                n_soft=len(soft_items), soft_app_id=soft_app_id, soft_pod_off=soft_pod_off, soft_pod_name=soft_pod_name,
                node_ids=node_ids)


def _directory(ids, size):
    d = np.full(max(size, 1), -1, np.int64)                  # one spare entry: indexing with max(id, 0) stays in bounds
    d[ids] = np.arange(len(ids))
    return d


def evaluate(enc: dict):
    """The per-call side over the encoded arrays, with numpy -> (overhead (cpu, mem, gpu), nonsched (cpu, mem, gpu),
    has_reservation uint8[n_pods], n_warned).  Raises OverflowError where gp_node_overhead returns GP_ERR_UNREPRESENTABLE."""
    node_id = np.asarray(enc["node_id"], np.int64)
    used = node_id >= 0
    listed = used & (np.asarray(enc["listed"], bool) if enc.get("listed") is not None else True)
    ak, ai, nm = (np.asarray(enc[k], np.int64) for k in ("app_key", "app_id", "name_id"))
    names = max(int(enc["n_names"]), 1)
    rr_of = _directory(np.asarray(enc["rr_app_key"], np.int64), int(enc["n_app_keys"]))
    soft_of = _directory(np.asarray(enc["soft_app_id"], np.int64), int(enc["n_app_ids"]))

    def members(off, name):
        seg = np.repeat(np.arange(len(off) - 1), np.diff(off))
        return seg * names + np.asarray(name, np.int64)

    labelled = listed & (ak >= 0)
    r = np.where(labelled, rr_of[np.where(labelled, ak, 0)], -1)    # fields of unlisted records and free slots are never read
    in_rr = (r >= 0) & np.isin(r * names + nm, members(np.asarray(enc["rr_pod_off"]), enc["rr_pod_name"]))
    s = np.where(labelled & np.asarray(enc["is_executor"], bool), soft_of[np.where(labelled, ai, 0)], -1)
    in_soft = (s >= 0) & np.isin(s * names + nm, members(np.asarray(enc["soft_pod_off"]), enc["soft_pod_name"]))
    has = labelled & (in_rr | in_soft)
    rows = _directory(np.asarray(enc["node_ids"], np.int64), int(enc["n_node_ids"]))
    row = np.where(used, rows[np.maximum(node_id, 0)], -1)
    counted = listed & ~has & (row >= 0)
    spark = np.asarray(enc["spark_scheduler"], bool)
    n_rows = len(enc["node_ids"])
    reqs = [np.asarray(enc[k], np.int64) if enc.get(k) is not None else np.zeros(len(node_id), np.int64)
            for k in ("req_cpu_milli", "req_mem_bytes", "req_gpu")]
    out = []
    for sel in (counted, counted & ~spark):
        triple = []
        for v in reqs:
            lo, hi = np.zeros(n_rows, np.int64), np.zeros(n_rows, np.int64)
            np.add.at(lo, row[sel], v[sel] & 0xFFFFFFFF)
            np.add.at(hi, row[sel], v[sel] >> 32)
            tot = [(int(h) << 32) + int(x) for h, x in zip(hi, lo)]
            if any(t >= _MAX for t in tot):
                raise OverflowError("a per-node sum >= 2^61")
            triple.append(np.array(tot, np.int64))
        out.append(tuple(triple))
    n_warned = int((counted & spark & (r >= 0)).sum())
    return out[0], out[1], has.astype(np.uint8), n_warned


def synthetic_cluster(seed: int, n_nodes: int, n_pods: int, big_apps: int = 0, big_executors: int = 2000, huge_app: int = 0,
                      absent_frac: float = 0.01):
    """A seeded cluster as the event side sees it: every pod goes through PodRecords.add; a fraction absent_frac of them is
    missing from the lister (deleted, delete event not yet seen).  Pods: ~3 non-spark pods per node (no labels, default
    scheduler, with init containers), then spark applications (driver + executors) across 16 namespaces until n_pods:
    `big_apps` of them with `big_executors` executors, one with `huge_app` executors if given, the rest 0-40 executors.
    Most applications have a ResourceReservation listing the driver and most executors (plus names of pods that are gone);
    some have soft reservations for extra executors; a few appIDs repeat across namespaces.
    -> (nodes, records, lister, rrs, soft, pods)"""
    rng = np.random.default_rng(seed)
    nodes = [f"node-{i}" for i in range(n_nodes)]
    records = PodRecords()
    lister, rrs, soft, pods = {}, {}, {}, []
    gib = 1 << 30
    node_of = rng.integers(0, n_nodes, n_pods)
    k = 0

    def emit(pod):
        nonlocal k
        pod["uid"] = f"uid-{k}"
        pod["nodeName"] = nodes[node_of[k]]
        k += 1
        pods.append(pod)
        records.add(pod)
        if rng.random() >= absent_frac:
            lister[(pod["namespace"], pod["name"])] = pod

    n_sys = min(n_pods, 3 * n_nodes)
    cpu = rng.integers(1, 500, n_sys)
    mem = rng.integers(1, 2048, n_sys) << 20
    for j in range(n_sys):
        emit({"namespace": "kube-system", "name": f"ds-{j}", "labels": {}, "schedulerName": "default-scheduler",
              "containers": [{"cpu": int(cpu[j]), "memory": int(mem[j])}],
              "initContainers": [{"cpu": int(cpu[j]) + 100 * (j % 3), "memory": 64 << 20}]})
    sizes = [huge_app] if huge_app else []
    sizes += [big_executors] * big_apps
    a = 0
    while k < n_pods:
        execs = sizes[a] if a < len(sizes) else int(rng.integers(0, 41))
        execs = min(execs, n_pods - k - 1)
        ns = f"ns-{a % 16}"
        app = f"app-{a // 2}" if a % 7 == 3 else f"app-{a}"      # every 7th application reuses an appID in another namespace
        gpu = int(rng.integers(0, 2))
        drv_labels = {SPARK_APP_ID_LABEL: app, SPARK_ROLE_LABEL: "driver"}
        exe_labels = {SPARK_APP_ID_LABEL: app, SPARK_ROLE_LABEL: EXECUTOR}
        sched = SPARK_SCHEDULER_NAME if a % 11 else "default-scheduler"
        names = [f"{app}-driver"] + [f"{app}-exec-{e}" for e in range(execs)]
        for e, name in enumerate(names):
            emit({"namespace": ns, "name": name, "labels": exe_labels if e else drv_labels, "schedulerName": sched,
                  "containers": [{"cpu": 1000 * (1 + e % 4), "memory": (1 + e % 8) * gib, "nvidia.com/gpu": gpu}]})
        kind = a % 5
        if kind != 4:                                              # a ResourceReservation: driver + most executors
            reserved = names[:1 + (execs * 3) // 4] + [f"{app}-exec-gone-{x}" for x in range(2)]
            rrs[(ns, app)] = reserved
        if kind in (1, 4) and execs:                               # soft reservations for the remaining executors
            soft.setdefault(app, []).extend(names[1 + (execs * 3) // 4:] + ([names[0]] if kind == 4 else []))
        a += 1
    return nodes, records, lister, rrs, soft, pods


# ---- the resident table (gp_overhead_table_*) -------------------------------------------------------------------------------
_FREE_ROW = (-1, 0, 0, 0, 0, -1, -1, 0, 0, 0)     # node_id, cpu, mem, gpu, listed, app_key, app_id, name_id, is_executor, spark
_ROW_COLS = (("node_id", np.int32), ("req_cpu_milli", np.int64), ("req_mem_bytes", np.int64), ("req_gpu", np.int64),
             ("listed", np.uint8), ("app_key", np.int32), ("app_id", np.int32), ("name_id", np.int32),
             ("is_executor", np.uint8), ("spark_scheduler", np.uint8))
_SIZE_KEYS = ("n_slots", "n_node_ids", "n_app_keys", "n_app_ids", "n_names")


class _CountedInterner:
    """Dense ids with reference counts: the id of a key whose last reference is released goes to the next new key."""

    def __init__(self):
        self.ids, self.count, self._free = {}, [], []

    def acquire(self, key) -> int:
        i = self.ids.get(key)
        if i is None:
            if self._free:
                i = self._free.pop()
            else:
                i = len(self.count)
                self.count.append(0)
            self.ids[key] = i
        self.count[i] += 1
        return i

    def release(self, key):
        i = self.ids[key]
        self.count[i] -= 1
        if not self.count[i]:
            del self.ids[key]
            self._free.append(i)

    @property
    def bound(self) -> int:
        """every id in use is below this"""
        return len(self.count)


class OverheadTable(PodRecords, ResidentTable):
    """The host side of the resident overhead table: PodRecords' slots (same numbering), the pod lister, the
    ResourceReservation cache and the soft store, kept as the shim's informer handlers see them, and turned into the deltas of
    gp_overhead_table_update.  Ids come from reference-counted interners over the slots' rows, the RR flags and the members,
    so the ids of nodes, apps and pod names that are gone are reused.

    Events: add / update / delete (the pod informer through the nodeName filter, as PodRecords), lister_set(pod) /
    lister_delete(namespace, name), rr_set((namespace, appID), Status.Pods values) / rr_delete, soft_set(appID, Reservations
    keys) / soft_delete.  delta() -> the arrays of one gp_overhead_table_update: what changed since the last delta (everything
    after a reset); see ResidentTable.  A request >= 2^61 is refused when it arrives."""

    name, writes = "overhead", ("slot", "rr_app_key", "member_kind")

    def __init__(self, n_slots=64, n_node_ids=64, n_app_keys=64, n_app_ids=64, n_names=64):
        PodRecords.__init__(self)
        ResidentTable.__init__(self, TableMirror(), n_slots=n_slots, n_node_ids=n_node_ids, n_app_keys=n_app_keys,
                               n_app_ids=n_app_ids, n_names=n_names)
        self.lister, self.rrs, self.soft = {}, {}, {}
        self._nodes, self._keys, self._apps, self._names = (_CountedInterner() for _ in range(4))
        self._row, self._refs = [], []                  # per slot: its row (ids), the interner references the row holds
        self._by_pod, self._pod_of = {}, {}              # (namespace, name) -> slots whose record names that pod, and back
        self._flags = set()                              # app key ids with a ResourceReservation
        self._members = {}                               # (kind, app, name) ids -> holders (0: absent)
        self._dirty, self._flag_touched, self._member_touched = {}, {}, {}   # -> what the device holds since the last delta

    # ---- pod records (PodRecords' add / update / delete land here)
    def _record(self, pod):
        super()._record(pod)
        self._refresh(self._at[(pod["nodeName"], pod["uid"])])

    def _remove(self, pod):
        at = self._at.get((pod["nodeName"], pod["uid"]))
        super()._remove(pod)
        if at is not None:
            self._refresh(at)

    # ---- the lister
    def lister_set(self, pod):
        key = (pod["namespace"], pod["name"])
        self.lister[key] = pod
        for at in list(self._by_pod.get(key, ())):
            self._refresh(at)

    def lister_delete(self, namespace, name):
        if self.lister.pop((namespace, name), None) is not None:
            for at in list(self._by_pod.get((namespace, name), ())):
                self._refresh(at)

    # ---- ResourceReservations and the soft store
    def rr_set(self, key, names):
        kid = self._keys.acquire(key)
        self._touch_flag(kid)
        self._flags.add(kid)
        self._hold(0, kid, names)
        self._drop_rr(key)
        self.rrs[key] = list(names)

    def rr_delete(self, key):
        if key in self.rrs:
            kid = self._keys.ids[key]
            self._touch_flag(kid)
            self._flags.discard(kid)
            self._drop_rr(key)

    def soft_set(self, app, names):
        aid = self._apps.acquire(app)
        self._hold(1, aid, names)
        self._drop_soft(app)
        self.soft[app] = list(names)

    def soft_delete(self, app):
        if app in self.soft:
            self._drop_soft(app)

    # ---- queries
    def node_ids(self, nodes) -> np.ndarray:
        """the table's ids of these node names; -1 for a node without one (it has no records: its overhead is zero)"""
        return np.array([self._nodes.ids.get(n, -1) for n in nodes], np.int32)

    def answer(self, nodes, query):
        """GetOverhead / GetNonSchedulableOverhead of `nodes` in their order through query(node_ids) -- a device query or
        evaluate(to_encoding(mirror, node_ids)) -- asked for the nodes that have an id; the others are zero.
        -> (overhead (cpu, mem, gpu), nonsched (cpu, mem, gpu), has_reservation, n_warned)"""
        ids = self.node_ids(nodes)
        known = ids >= 0
        ov, ns, has, warned = query(ids[known])
        cols = [np.zeros(len(nodes), np.int64) for _ in range(6)]
        for c, v in zip(cols, tuple(ov) + tuple(ns)):
            c[known] = v
        return tuple(cols[:3]), tuple(cols[3:]), has, warned

    # ---- internals
    def _bounds(self):
        return dict(n_slots=len(self.slots), n_node_ids=self._nodes.bound, n_app_keys=self._keys.bound,
                    n_app_ids=self._apps.bound, n_names=self._names.bound)

    def _changes(self, replay):
        if replay:
            slots = [at for at, row in enumerate(self._row) if row != _FREE_ROW]
            flags = sorted(self._flags)
            members = sorted(t for t, n in self._members.items() if n)
        else:
            slots = sorted(at for at, was in self._dirty.items() if self._row[at] != was)
            flags = sorted(k for k, was in self._flag_touched.items() if (k in self._flags) != was)
            members = sorted(t for t, was in self._member_touched.items() if (self._members.get(t, 0) > 0) != was)
        rows = [self._row[at] for at in slots]
        d = {"slot": np.array(slots, np.int32)}
        for j, (name, t) in enumerate(_ROW_COLS):
            d[name] = np.array([r[j] for r in rows], t)
        d["rr_app_key"] = np.array(flags, np.int32)
        d["rr_exists"] = np.array([k in self._flags for k in flags], np.uint8)
        d["member_kind"] = np.array([t[0] for t in members], np.uint8)
        d["member_app"] = np.array([t[1] for t in members], np.int32)
        d["member_name"] = np.array([t[2] for t in members], np.int32)
        d["member_present"] = np.array([self._members.get(t, 0) > 0 for t in members], np.uint8)
        self._dirty, self._flag_touched, self._member_touched = {}, {}, {}
        return d

    def _refresh(self, at):
        while len(self._row) < len(self.slots):
            self._row.append(_FREE_ROW)
            self._refs.append(())
        rec = self.slots[at]
        refs, row = [], _FREE_ROW

        def acquire(interner, key):
            refs.append((interner, key))
            return interner.acquire(key)

        if rec is not None:
            ns, name, node, req = rec
            pod = self.lister.get((ns, name))
            if pod is None:
                row = (acquire(self._nodes, node),) + tuple(req) + (0, -1, -1, 0, 0, 0)
            else:
                labels = pod.get("labels") or {}
                app = labels.get(SPARK_APP_ID_LABEL)
                ak, ai = (-1, -1) if app is None else (acquire(self._keys, (pod["namespace"], app)), acquire(self._apps, app))
                row = (acquire(self._nodes, node),) + tuple(req) + (
                    1, ak, ai, acquire(self._names, pod["name"]), int(labels.get(SPARK_ROLE_LABEL) == EXECUTOR),
                    int(pod.get("schedulerName") == SPARK_SCHEDULER_NAME))
        for interner, key in self._refs[at]:
            interner.release(key)
        old = self._row[at]
        self._dirty.setdefault(at, old)
        self._row[at], self._refs[at] = row, tuple(refs)
        self._index(at, self._pod_of.get(at), None if rec is None else (rec[0], rec[1]))

    def _index(self, at, old_pod, new_pod):
        if old_pod == new_pod:
            return
        if old_pod is not None:
            self._by_pod[old_pod].discard(at)
            if not self._by_pod[old_pod]:
                del self._by_pod[old_pod]
            del self._pod_of[at]
        if new_pod is not None:
            self._by_pod.setdefault(new_pod, set()).add(at)
            self._pod_of[at] = new_pod

    def _touch_flag(self, kid):
        self._flag_touched.setdefault(kid, kid in self._flags)

    def _hold(self, kind, app, names):
        """one holder of (kind, app, name) per distinct name (Status.Pods values may repeat); each holds a name id"""
        for name in dict.fromkeys(names):
            t = (kind, app, self._names.acquire(name))
            self._member_touched.setdefault(t, self._members.get(t, 0) > 0)
            self._members[t] = self._members.get(t, 0) + 1

    def _release(self, kind, app, names):
        for name in dict.fromkeys(names):
            t = (kind, app, self._names.ids[name])
            self._member_touched.setdefault(t, self._members[t] > 0)
            self._members[t] -= 1
            if not self._members[t]:
                del self._members[t]
            self._names.release(name)

    def _drop_rr(self, key):
        old = self.rrs.pop(key, None)
        if old is not None:
            self._release(0, self._keys.ids[key], old)
            self._keys.release(key)

    def _drop_soft(self, app):
        old = self.soft.pop(app, None)
        if old is not None:
            self._release(1, self._apps.ids[app], old)
            self._apps.release(app)


class TableMirror:
    """What gp_overhead_table_update leaves on the device, with numpy: apply(delta) in the order the library would, so
    evaluate(to_encoding(mirror, node_ids)) is the device's answer without a device."""

    def __init__(self):
        self.size = None

    def apply(self, d: dict):
        if d.get("reset"):
            self.size = dict(d["reset"])
            n = self.size["n_slots"]
            self.cols = {name: np.full(n, free, t) for (name, t), free in zip(_ROW_COLS, _FREE_ROW)}
            self.rr = np.zeros(self.size["n_app_keys"], np.uint8)
            self.members = set()
        s = np.asarray(d["slot"], np.int64)
        for name, t in _ROW_COLS:
            v = d.get(name)
            default = {"listed": 1, "req_gpu": 0, "is_executor": 0, "spark_scheduler": 0}.get(name)
            self.cols[name][s] = np.asarray(v, t) if v is not None else default
        self.rr[np.asarray(d["rr_app_key"], np.int64)] = np.asarray(d["rr_exists"], np.uint8) != 0
        for k, a, nm, p in zip(*(np.asarray(d[x]).tolist() for x in ("member_kind", "member_app", "member_name", "member_present"))):
            (self.members.add if p else self.members.discard)((k, a, nm))


def to_encoding(mirror: TableMirror, node_ids) -> dict:
    """The gp_node_overhead arrays of the table's state: its slots, rr_app_key = the app keys whose RR flag is set with their
    kind-0 members, soft_app_id = the app ids with kind-1 members."""
    by = ({}, {})
    for k, a, nm in sorted(mirror.members):
        by[k].setdefault(a, []).append(nm)
    rr_keys = [int(k) for k in np.nonzero(mirror.rr)[0]]
    rr_names = [by[0].get(k, []) for k in rr_keys]
    soft_ids = sorted(by[1])
    soft_names = [by[1][a] for a in soft_ids]

    def csr(lists):
        off = np.zeros(len(lists) + 1, np.int64)
        np.cumsum([len(x) for x in lists], out=off[1:])
        return off, np.array([v for x in lists for v in x], np.int32)

    rr_off, rr_name = csr(rr_names)
    soft_off, soft_name = csr(soft_names)
    enc = {name: mirror.cols[name].copy() for name, _ in _ROW_COLS}
    enc.update(n_pods=mirror.size["n_slots"], **{k: mirror.size[k] for k in _SIZE_KEYS[1:]},
               n_rr=len(rr_keys), rr_app_key=np.array(rr_keys, np.int32), rr_pod_off=rr_off, rr_pod_name=rr_name,
               n_soft=len(soft_ids), soft_app_id=np.array(soft_ids, np.int32), soft_pod_off=soft_off, soft_pod_name=soft_name,
               node_ids=np.asarray(node_ids, np.int32))
    return enc
