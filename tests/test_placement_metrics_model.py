"""The closed form behind gp_placement_metrics (distinct executor nodes, driver membership, and
cross = T*S - (S^2 + sum c_z^2) / 2 over the metric-zone pod histogram) against the literal, string-keyed restatement of
ReportInitialDriverExecutorCollocationMetric, ReportInitialNodeCountMetrics and ReportCrossZoneMetric with Go map semantics:
random rows and the corner cases, every zone-map iteration order giving the same cross-zone count."""
import itertools

import numpy as np

import placement_metrics_ref as ref


def _cluster(rng, n, n_labels, missing=0.1, literal_unknown=True):
    names = ["node-%05d" % v for v in range(n)]
    labels = []
    for v in range(n):
        r = rng.random()
        if r < missing:
            labels.append({})
        elif literal_unknown and r < 2 * missing:
            labels.append({ref.LABEL_ZONE_FAILURE_DOMAIN: "unknown-zone"})
        else:
            labels.append({ref.LABEL_ZONE_FAILURE_DOMAIN: "zone-%d" % rng.integers(0, n_labels), "other": "x"})
    return names, labels


def _rows(rng, n, q, kmax, placed_frac=0.8):
    count = rng.integers(0, kmax + 1, q).astype(np.int32)
    off = np.zeros(q + 1, np.int64)
    np.cumsum(count, out=off[1:])
    driver = np.where(rng.random(q) < placed_frac, rng.integers(0, n, q), -1).astype(np.int32)
    execn = rng.integers(0, n, int(off[-1])).astype(np.int32)
    return driver, execn, off, count


def _check(driver, execn, off, count, names, labels, ig=None, group=None, rng=None):
    zone, _ = ref.intern_metric_zones(labels)
    want = np.asarray(ref.literal_batch(driver, execn, off, count, names, labels, ig, group, rng), np.int64).reshape(-1, 6)
    got = ref.closed_form(driver, execn, off, count, zone, ig, group)
    assert np.array_equal(got, want)


def test_random_rows_match_literal():
    rng = np.random.default_rng(11)
    for n, n_labels, kmax in ((5, 2, 6), (40, 3, 12), (300, 7, 40)):
        names, labels = _cluster(rng, n, n_labels)
        _check(*_rows(rng, n, 200, kmax), names, labels, rng=rng)


def test_instance_group_scope_matches_literal():
    """nodes outside the row's availableNodes count in T and in no zone"""
    rng = np.random.default_rng(12)
    n = 120
    names, labels = _cluster(rng, n, 4)
    ig = rng.integers(-1, 3, n).astype(np.int32)
    driver, execn, off, count = _rows(rng, n, 150, 10)
    group = rng.integers(0, 3, len(driver)).astype(np.int32)
    _check(driver, execn, off, count, names, labels, ig, group, rng)


def test_corner_cases():
    names = ["a", "b", "c", "d"]
    z = ref.LABEL_ZONE_FAILURE_DOMAIN
    labels = [{z: "z1"}, {z: "z2"}, {}, {z: "unknown-zone"}]
    cases = [
        (0, []),                      # empty ExecutorNodes: no-collocation, execs_per_node -1, one pod
        (1, [1, 1, 1]),               # every executor on the driver's node
        (0, [0, 1, 0]),               # the driver among the executors
        (1, [0, 1, 2, 0, 1, 2]),      # nodes repeated across rounds
        (2, [3, 2]),                  # a missing label next to a node labelled unknown-zone: one zone
    ]
    driver = np.array([d for d, _ in cases], np.int32)
    count = np.array([len(e) for _, e in cases], np.int32)
    off = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
    execn = np.array([v for _, e in cases for v in e], np.int32)
    zone, nz = ref.intern_metric_zones(labels)
    assert nz == 3 and zone[2] == zone[3]
    got = ref.closed_form(driver, execn, off, count, zone)
    assert [tuple(r) for r in got] == [(0, 0, -1, 1, 0, 0), (1, 1, 3, 1, 0, 6), (2, 2, 1, 2, 3, 6), (2, 3, 2, 3, 16, 21),
                                       (2, 2, 1, 1, 0, 3)]
    _check(driver, execn, off, count, names, labels)


def test_every_node_its_own_zone():
    rng = np.random.default_rng(13)
    n = 64
    names = ["n%d" % v for v in range(n)]
    labels = [{ref.LABEL_ZONE_FAILURE_DOMAIN: "z%d" % v} for v in range(n)]
    _check(*_rows(rng, n, 100, 30), names, labels, rng=rng)


def test_cross_zone_traffic_independent_of_map_order():
    counts = {"a": 3, "b": 1, "c": 7, "d": 2}
    T = sum(counts.values()) + 4                 # four pods outside every zone
    vals = set()
    for perm in itertools.permutations(counts):
        vals.add(ref.cross_zone_traffic({z: counts[z] for z in perm}, T))
    S, sq = sum(counts.values()), sum(c * c for c in counts.values())
    assert vals == {T * S - (S * S + sq) // 2}


def test_large_T_fits_int64():
    """T near 2^24 (the exe_count bound): the closed form is exact in int64 and equals the literal"""
    k = (1 << 24) - 1
    rng = np.random.default_rng(14)
    n = 50
    zone_of = rng.integers(0, 5, n)
    execn = rng.integers(0, n, k).astype(np.int32)
    zone = zone_of.astype(np.int32)
    got = ref.closed_form(np.array([3], np.int32), execn, np.array([0, k], np.int64), np.array([k], np.int32), zone)[0]
    T = k + 1
    c = np.bincount(zone_of[np.append(execn, 3)], minlength=5).astype(object)
    hist = {z: int(c[z]) for z in range(5) if c[z]}
    assert got[4] == ref.cross_zone_traffic(hist, T) and got[5] == T * (T - 1) // 2
    assert got[5] < 2 ** 63 and T * T < 2 ** 63
