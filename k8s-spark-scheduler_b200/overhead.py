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
