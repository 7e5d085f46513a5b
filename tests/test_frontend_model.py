"""frontend_ref (the front end in Python integers, which the GPU tests compare the kernels with) pinned to the evidence the
project already has: the golden vectors of the reference's own sorter tests, the literal C oracle and the pure-Python
restatement.  No GPU."""
import numpy as np

import frontend_ref as fr
from helpers import case_arrays


def _ids(names, zones):
    """dense zone ids in first-seen order, n_zones, name ranks"""
    zid, seen = [], {}
    for n in names:
        zid.append(seen.setdefault(zones.get(n, "default"), len(seen)))
    order = sorted(range(len(names)), key=lambda i: names[i])
    rank = [0] * len(names)
    for r, i in enumerate(order):
        rank[i] = r
    return zid, max(len(seen), 1), rank


def test_golden_sort_and_label_cases(golden):
    for case in golden["sort_cases"]:
        names, cpu, mem, _ = case_arrays(case["nodes"])
        zid, nz, rank = _ids(names, case["zones"])
        d, e = fr.potential_nodes(cpu.tolist(), mem.tolist(), zid, nz, rank)
        assert [names[i] for i in d] == case["expect_priority_order"], case["id"]
        assert [names[i] for i in e] == case["expect_priority_order"], case["id"]
    for case in golden["label_cases"]:
        names = case["input"]
        n = len(names)
        zid, nz, rank = _ids(names, {})
        lr = [case["rank"].get(nm, -1) for nm in names]
        d, e = fr.potential_nodes([1] * n, list(range(1, n + 1)), zid, nz, rank, lr_d=lr, lr_e=lr)
        assert [names[i] for i in d] == case["expect"] and [names[i] for i in e] == case["expect"], case["id"]


def _random_sort_case(rng, n):
    names = ["node-%05d" % int(x) for x in rng.permutation(n * 3)[:n]]
    cpu = (rng.integers(-2, 6, n) * 1000).tolist()
    mem = (rng.integers(-1, 5, n) * (1 << 30)).tolist()
    zones = {nm: "zone-%d" % rng.integers(0, 4) for nm in names} if rng.random() < 0.6 else {}
    unsched = (rng.random(n) < 0.1).astype(np.uint8)
    ready = (rng.random(n) < 0.9).astype(np.uint8)
    cand = (rng.random(n) < 0.6).astype(np.uint8)
    lr_d = rng.integers(-1, 3, n).astype(np.int32) if rng.random() < 0.5 else None
    lr_e = rng.integers(-1, 2, n).astype(np.int32) if rng.random() < 0.5 else None
    return names, cpu, mem, zones, unsched, ready, cand, lr_d, lr_e


def test_potential_nodes_matches_the_oracles(oracle):
    """300 random in-range clusters (heavy ties, negative values, zones, masks, labels): frontend_ref == the literal C oracle
    == oracle/pyref.py.  Clusters whose zone totals tie are skipped: the reference leaves their zone order open."""
    from oracle import pyref
    rng = np.random.default_rng(0xF1)
    compared = 0
    for trial in range(300):
        n = int(rng.integers(1, 80))
        names, cpu, mem, zones, unsched, ready, cand, lr_d, lr_e = _random_sort_case(rng, n)
        zid, nz, rank = _ids(names, zones)
        if fr.zone_totals_tied(cpu, mem, zid, nz):
            continue
        compared += 1
        d, e = fr.potential_nodes(cpu, mem, zid, nz, rank, cand, unsched, ready, lr_d, lr_e)
        cl = oracle.Cluster(names, cpu, mem, np.zeros(n, np.int64), zone=[zones.get(nm, "default") for nm in names],
                            unschedulable=unsched, ready=ready)
        cand_names = [nm for nm, m in zip(names, cand) if m]
        wd, we = cl.potential_nodes(cand_names, lr_d, lr_e)
        assert [names[i] for i in d] == wd and [names[i] for i in e] == we, trial
        meta = {names[i]: (cpu[i], mem[i], 0) for i in range(n)}
        rk = lambda lr: None if lr is None else {names[i]: int(lr[i]) for i in range(n) if lr[i] >= 0}
        pd, pe = pyref.potential_nodes(meta, zones, cand_names, {names[i] for i in range(n) if unsched[i]},
                                       {names[i] for i in range(n) if not ready[i]}, rk(lr_d), rk(lr_e))
        assert [names[i] for i in d] == pd and [names[i] for i in e] == pe, trial
    assert compared > 150


def test_availability_matches_the_oracles(oracle):
    """random node tables and reservations (rows off the table, all-zero rows, negative allocatable, overhead above
    allocatable): avail and sched == the C oracle's NodeSchedulingMetadataForNodes and pyref's, the first-fit
    availability == the C oracle's rescheduleExecutor availability (overhead twice where the usage map has an entry)."""
    from oracle import pyref
    rng = np.random.default_rng(0xF2)
    for trial in range(200):
        n, R = int(rng.integers(1, 40)), int(rng.integers(0, 120))
        names = ["node-%05d" % i for i in range(n)]
        alloc = [rng.integers(-4, 97, n) * 1000, rng.integers(-2, 385, n) * (1 << 30), rng.integers(0, 9, n)]
        over = [rng.integers(0, 200, n) * 1000, rng.integers(0, 4, n) * (1 << 28), rng.integers(0, 2, n)]
        rnode = rng.integers(-1, n, R).astype(np.int32)
        res = [rng.integers(0, 8, R) * 500, rng.integers(0, 16, R) * (1 << 29), rng.integers(0, 2, R)]
        zero = rng.random(R) < 0.3                                  # reservations whose resources are all zero
        res = [np.where(zero, 0, x) for x in res]
        ov = over if trial % 3 else None
        av, sc, ff = fr.availability(alloc, ov, rnode, res)
        rn = [names[i] if i >= 0 else "gone" for i in rnode]
        wav, wsc = oracle.node_scheduling_metadata(names, alloc, ov, rn, res)
        wff = oracle.reschedule_available(names, alloc, ov, rn, res)
        for d in range(3):
            assert av[d] == wav[d].tolist() and sc[d] == wsc[d].tolist() and ff[d] == wff[d].tolist(), (trial, d)
        t = lambda cols, i: tuple(int(c[i]) for c in cols)
        pav, psc = pyref.node_scheduling_metadata({names[i]: t(alloc, i) for i in range(n)},
                                                  {names[i]: t(ov, i) for i in range(n)} if ov else {},
                                                  [(rn[r], t(res, r)) for r in range(R)])
        for i in range(n):
            assert pav[names[i]] == t(av, i) and psc[names[i]] == t(sc, i), (trial, i)


def test_unbounded_and_ties():
    big = (1 << 61) - 1
    av, sc, ff = fr.availability(([big], [-big], [0]), ([-big], [big], [0]), [0, 0, 5, -1], ([-big, -big, 1, 1], [big, big, 1, 1], [0] * 4))
    assert av[0] == [4 * big] and av[1] == [-4 * big] and sc[0] == [2 * big] and ff[0] == [5 * big] and ff[1] == [-5 * big]
    assert fr.in_domain(big) and fr.in_domain(-big) and not fr.in_domain(big + 1) and not fr.in_domain(-big - 1)
    # four nodes near 2^61 in one zone: the total is exact, the zone sorts last
    cpu, mem, zid = [0] * 5, [big] * 4 + [5], [0, 0, 0, 0, 1]
    assert fr.zone_priority(cpu, mem, zid, 3) == [2, 1, 0]           # zone 2 has no node: total (0, 0)
    assert fr.priority_order(cpu, mem, zid, 3) == [4, 0, 1, 2, 3]
    assert fr.zone_totals_tied([1, 1], [2, 2], [0, 1], 2) and not fr.zone_totals_tied([1, 2], [2, 2], [0, 1], 2)
    keys = fr.node_keys([1, 1, 1, 2], [7, 7, 7, 7])
    assert fr.undefined_ties([0, 1, 2, 3], keys, [0, 1, 1, 5]) == 1 and fr.undefined_ties([0, 1, 2, 3], keys, None) == 0
    assert fr.label_sort([3, 1, 2, 0], [0, -1, 0, 5]) == [2, 0, 3, 1]     # ranks 5, -1, 0, 0: stable, unknown last
