"""A literal, string-keyed restatement of the three placement reporters selectDriverNode calls after a successful pack
(internal/extender/resource.go:352-357), and a numpy form of the closed form the device computes.

literal(): ReportInitialDriverExecutorCollocationMetric (internal/metrics/metrics.go:223-252), ReportInitialNodeCountMetrics
(:254-275) and ReportCrossZoneMetric + crossZoneTraffic (:277-318, 322-330) over node NAMES and label maps, with Go's map
semantics: the zone map is iterated in a random order (`rng`), a missing failure-domain label becomes "unknown-zone", and
integer division truncates.  It returns the values the reporters emit, as one record per application."""
import numpy as np

LABEL_ZONE_FAILURE_DOMAIN = "failure-domain.beta.kubernetes.io/zone"
NOT_REPORTED = (-1, 0, 0, 0, 0, 0)
FIELDS = ("collocation", "distinct_exec_nodes", "execs_per_node", "n_zones", "cross_zone_pairs", "total_pairs")


def cross_zone_traffic(num_pods_per_zone: dict, total_num_pods: int, rng=None) -> int:
    """metrics.go:322-330, iterating the map in a random order as Go does"""
    zones = list(num_pods_per_zone)
    if rng is not None:
        rng.shuffle(zones)
    num_pods_in_different_zone = total_num_pods
    traffic = 0
    for z in zones:
        n = num_pods_per_zone[z]
        num_pods_in_different_zone -= n
        traffic += n * num_pods_in_different_zone
    return traffic


def literal(driver_node_name: str, executor_node_names: list, available_nodes: dict, rng=None) -> tuple:
    """One application: available_nodes = {name: labels dict} (the Predicate's availableNodes; a lister's names are unique, so
    visiting the nodes that host pods is the reference's walk over every node restricted to those it keeps).  -> FIELDS"""
    executor_set = {n: True for n in executor_node_names}                       # toExecutorNodeNamesSet
    if not executor_set.get(driver_node_name, False):
        collocation = 0                                                          # "no-collocation"
    elif len(executor_set) == 1:
        collocation = 1                                                          # "driver-collocated-with-all-executors"
    else:
        collocation = 2                                                          # "driver-collocated-with-some-executors"
    executor_count = len(executor_node_names)
    if executor_count == 0:                                                      # ReportInitialNodeCountMetrics returns
        execs_per_node = -1
    else:
        execs_per_node = int(executor_count / len(executor_set))                 # Go int division (both positive)
    num_pods_per_node = {driver_node_name: 1}
    for n in executor_node_names:
        num_pods_per_node[n] = num_pods_per_node.get(n, 0) + 1
    num_pods_per_zone = {}
    for name, num_pods in num_pods_per_node.items():
        labels = available_nodes.get(name)
        if labels is not None:
            zone = labels.get(LABEL_ZONE_FAILURE_DOMAIN, "unknown-zone")
            num_pods_per_zone[zone] = num_pods_per_zone.get(zone, 0) + num_pods
    total = executor_count + 1
    return (collocation, len(executor_set), execs_per_node, len(num_pods_per_zone),
            cross_zone_traffic(num_pods_per_zone, total, rng), total * (total - 1) // 2)


def literal_batch(driver, execn, off, count, names, labels, instance_group=None, group=None, rng=None):
    """literal() per row over node-index arrays: names[v] / labels[v] describe node v; row i's availableNodes are the nodes
    of its instance group (instance_group None: every node).  driver < 0 -> NOT_REPORTED."""
    avail = {}
    for v in range(len(names)):
        g = -2 if instance_group is None else int(instance_group[v])
        avail.setdefault(g, {})[names[v]] = labels[v]
    out = []
    for i, d in enumerate(driver):
        if d < 0:
            out.append(NOT_REPORTED)
            continue
        ex = [names[v] for v in execn[off[i]:off[i] + count[i]]]
        g = -2 if instance_group is None else (0 if group is None else int(group[i]))
        out.append(literal(names[d], ex, avail.get(g, {}), rng))
    return out


def intern_metric_zones(labels):
    """the metric zone column: the failure-domain label, a missing one interned as "unknown-zone" -> (ids, n_zones)"""
    ids, table = [], {}
    for lb in labels:
        ids.append(table.setdefault(lb.get(LABEL_ZONE_FAILURE_DOMAIN, "unknown-zone"), len(table)))
    return np.asarray(ids, np.int32), len(table)


def closed_form(driver, execn, off, count, zone, instance_group=None, group=None) -> np.ndarray:
    """The device's computation in numpy (int64, exact): per row the distinct executor nodes, the driver's membership and the
    pod histogram over the metric zones, cross = T*S - (S^2 + sum c^2) / 2.  -> int64 array [n_apps, 6] in FIELDS order."""
    driver = np.asarray(driver); zone = np.asarray(zone, np.int64)
    out = np.zeros((len(driver), 6), np.int64)
    out[:, 0] = -1
    for i, d in enumerate(driver):
        if d < 0:
            continue
        k = int(count[i])
        e = np.asarray(execn[off[i]:off[i] + k], np.int64)
        uniq = np.unique(e)
        distinct = len(uniq)
        hosts = bool(k) and bool(np.any(e == d))
        pods = np.append(e, d)
        if instance_group is not None:
            g = 0 if group is None else group[i]
            pods = pods[np.asarray(instance_group)[pods] == g]
        c = np.bincount(zone[pods]) if len(pods) else np.zeros(0, np.int64)
        c = c[c > 0].astype(np.int64)
        T, S = k + 1, int(c.sum())
        out[i] = (0 if not hosts else 1 if distinct == 1 else 2, distinct, k // distinct if k else -1, len(c),
                  T * S - (S * S + int((c * c).sum())) // 2, T * (T - 1) // 2)
    return out


def records_to_rows(rec) -> np.ndarray:
    """a PLACEMENT_DTYPE array -> int64 [n, 6] in FIELDS order"""
    return np.stack([np.asarray(rec[f], np.int64) for f in FIELDS], axis=1) if len(rec) else np.zeros((0, 6), np.int64)
