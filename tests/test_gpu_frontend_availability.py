"""Availability from reservations (gp_usage_scatter, gp_availability) against frontend_ref's sums over Python integers, and
the exact-int64 domain at this door.  Through gp_build_availability, gp_build_reschedule_availability, gp_prepare_cluster,
gp_prepare_cluster_zones and gp_reschedule_from_reservations the contract is the same: the exact result, or
GP_ERR_UNREPRESENTABLE -- never a wrapped or out-of-domain snapshot, whatever the wrapped value looks like; a refused call
leaves the context's snapshot as it was.  Zone totals have no domain: they are compared exactly."""
import numpy as np
import pytest

import frontend_ref as fr

pytestmark = pytest.mark.gpu

I64, I32 = np.int64, np.int32
B = 1 << 61
UNREPRESENTABLE = 6


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def _cols(t, n):
    return None if t is None else tuple(None if c is None else np.asarray(c, I64) for c in t)


def _refused(gangpack, fn):
    """fn's result, or None when the library refused with GP_ERR_UNREPRESENTABLE (any other error fails the test)"""
    try:
        return fn()
    except gangpack.native.GangpackError as e:
        assert e.status == UNREPRESENTABLE, e
        return None


def check_entries(gangpack, p, alloc, over, rnode, res, tag=""):
    """the five entries on one input.  For each: refused exactly when an input, a reservation sum or one of ITS results lies
    outside the domain, otherwise equal to frontend_ref.  -> the set of entries that refused"""
    n = len(alloc[0])
    rnode = np.asarray(rnode, I32)
    av, sc, ff = fr.availability(alloc, over, rnode, res)
    usage = fr.usage_sums(n, rnode, res)
    counted = [r for r, x in enumerate(rnode.tolist()) if 0 <= x < n]
    inputs = [int(v) for t in (alloc, over) if t is not None for c in t if c is not None for v in c]
    inputs += [int(c[r]) for c in res if c is not None for r in counted]
    flat = lambda t: [v for c in t for v in c]
    base_ok = all(map(fr.in_domain, inputs + flat(usage) + flat(av) + flat(sc)))
    ff_ok = base_ok and all(map(fr.in_domain, flat(ff)))
    alloc, over, res = _cols(alloc, n), _cols(over, n), _cols(res, len(rnode))
    refused = set()

    def outcome(name, ok, fn, check):
        got = _refused(gangpack, fn)
        if got is None:
            refused.add(name)
            assert not ok, (tag, name, "refused an input whose results are all representable")
        else:
            assert ok, (tag, name, "accepted an input with an unrepresentable quantity, sum or result")
            check(got)

    def same(got, want, dims=3):
        for d in range(dims):
            assert got[d].tolist() == want[d], (tag, d)

    outcome("gp_build_availability", base_ok, lambda: p.build_availability(alloc, over, rnode, res),
            lambda g: (same(g[0], av), same(g[1], sc)))
    outcome("gp_build_reschedule_availability", ff_ok, lambda: p.build_reschedule_availability(alloc, over, rnode, res),
            lambda g: same(g, ff))
    outcome("gp_prepare_cluster", base_ok, lambda: (p.prepare_cluster(alloc, over, rnode, res), p.get_snapshot())[1],
            lambda g: same(g, av))
    outcome("gp_prepare_cluster_zones", base_ok,
            lambda: (p.prepare_cluster_zones(alloc, over, rnode, res, layout=False), p.get_snapshot())[1], lambda g: same(g, av))
    # first fit of a zero request: the first node of the executor order whose first-fit availability is non-negative
    order = fr.priority_order(av[0], av[1])
    want = next((i for i in order if min(ff[0][i], ff[1][i], ff[2][i]) >= 0), -1) if ff_ok else None
    outcome("gp_reschedule_from_reservations", ff_ok,
            lambda: p.reschedule_from_reservations(alloc, over, rnode, res, (np.zeros(1, I64), np.zeros(1, I64)))[0],
            lambda g: g[0] == want or pytest.fail(f"{tag}: first fit {g[0]} != {want}"))
    return refused


# ---- sizes, rows off the table, the has-entry rule ---------------------------------------------------------------------

@pytest.mark.parametrize("n,R", [(1, 0), (1, 1), (255, 255), (256, 256), (257, 257), (256, 1), (257, 0), (50000, 257), (50000, 1000000)])
def test_sizes(gangpack, packer, n, R):
    rng = np.random.default_rng(n + R)
    alloc = (rng.integers(-4, 97, n) * 1000, rng.integers(-2, 385, n) * (1 << 30), rng.integers(0, 9, n))
    over = (rng.integers(0, 120, n) * 1000, rng.integers(0, 4, n) * (1 << 28), rng.integers(0, 2, n))   # often above allocatable
    rnode = rng.integers(-1, n + 1, R).astype(I32)                          # -1 and n: not in the table
    if R > 2:
        rnode[:2] = (2**31 - 1, -2**31)
    res = [rng.integers(0, 8, R) * 500, rng.integers(0, 16, R) * (1 << 29), rng.integers(0, 2, R)]
    zero = rng.random(R) < 0.2
    res = tuple(np.where(zero, 0, x) for x in res)
    assert check_entries(gangpack, packer, alloc, over, rnode, res, f"n={n} R={R}") == set()


def test_every_row_on_one_node(gangpack, packer):
    n, R = 257, 100000
    rng = np.random.default_rng(5)
    alloc = (np.full(n, 1 << 50, I64), np.full(n, 1 << 58, I64), np.full(n, 1 << 20, I64))
    res = (rng.integers(0, 1 << 30, R), rng.integers(0, 1 << 40, R), rng.integers(0, 4, R))
    assert check_entries(gangpack, packer, alloc, None, np.full(R, 256, I32), res) == set()


def test_zero_reservation_doubles_the_overhead(gangpack, packer):
    """a reservation whose resources are all zero still gives its node an entry in the usage map: the first-fit availability
    counts that node's overhead twice, and its neighbours' once"""
    n = 300
    alloc = (np.full(n, 8000, I64), np.full(n, 32 << 30, I64), np.full(n, 4, I64))
    over = (np.full(n, 500, I64), np.full(n, 1 << 30, I64), np.ones(n, I64))
    rnode = np.array([0, 255, 256, 299, n], I32)
    res = (np.zeros(5, I64), np.zeros(5, I64), np.zeros(5, I64))
    assert check_entries(gangpack, packer, alloc, over, rnode, res) == set()
    ff = packer.build_reschedule_availability(alloc, over, rnode, res)
    assert [int(ff[0][i]) for i in (0, 1, 254, 255, 256, 257, 298, 299)] == [7000, 7500, 7500, 7000, 7000, 7500, 7500, 7000]


@pytest.mark.parametrize("absent", ["alloc_gpu", "overhead_gpu", "res_gpu", "overhead_cpu", "overhead_mem", "all three gpu"])
def test_optional_columns(gangpack, packer, absent):
    n, R = 257, 600
    rng = np.random.default_rng(8)
    alloc = [rng.integers(1, 97, n) * 1000, rng.integers(1, 385, n) * (1 << 30), rng.integers(0, 9, n)]
    over = [rng.integers(0, 3, n) * 250, rng.integers(0, 4, n) * (1 << 28), rng.integers(0, 2, n)]
    res = [rng.integers(0, 8, R) * 500, rng.integers(0, 16, R) * (1 << 29), rng.integers(0, 2, R)]
    if absent in ("alloc_gpu", "all three gpu"): alloc[2] = None
    if absent in ("overhead_gpu", "all three gpu"): over[2] = None
    if absent in ("res_gpu", "all three gpu"): res[2] = None
    if absent == "overhead_cpu": over[0] = None
    if absent == "overhead_mem": over[1] = None
    assert check_entries(gangpack, packer, alloc, over, rng.integers(-1, n, R).astype(I32), res, absent) == set()


# ---- the domain lattice ----------------------------------------------------------------------------------------------------

def _lattice():
    """name -> (alloc, overhead, res_node, res) on 3 nodes, the quantity of interest in the cpu or memory column of node 1"""
    z3 = [0, 0, 0]

    def at(v, dim):                                         # a node column triple with v on node 1 in dimension dim
        t = [list(z3), list(z3), list(z3)]
        t[dim][1] = v
        return t

    def rows(vals, dim, node=1):
        t = [[0] * len(vals) for _ in range(3)]
        t[dim] = list(vals)
        return [node] * len(vals), t

    L = {}
    for dim, dn in ((0, "cpu"), (1, "mem"), (2, "gpu")):
        for v, vn in ((B - 1, "2^61-1"), (B, "2^61"), (-B + 1, "-2^61+1"), (-B, "-2^61"), ((1 << 63) - 1, "2^63-1"), (-(1 << 63), "-2^63")):
            L[f"alloc {dn} = {vn}"] = (at(v, dim), None, [], [[], [], []])
            L[f"overhead {dn} = {vn}"] = (at(0, dim), at(v, dim), [], [[], [], []])
            L[f"one reservation {dn} = {vn}"] = (at(0, dim), None, *rows([v], dim))
            L[f"one reservation {dn} = {vn} on a node off the table"] = (at(0, dim), None, *rows([v], dim, node=3))
    for dim, dn in ((0, "cpu"), (1, "mem")):
        # every input inside, the result just inside / just outside
        L[f"{dn}: alloc 2^61-1, reservation 0"] = (at(B - 1, dim), None, *rows([0], dim))
        L[f"{dn}: alloc 2^61-1, reservation -1 (avail 2^61)"] = (at(B - 1, dim), None, *rows([-1], dim))
        L[f"{dn}: alloc -2^61+1, reservation 1 (avail -2^61)"] = (at(-B + 1, dim), None, *rows([1], dim))
        L[f"{dn}: alloc -2^61+1, overhead 1 (sched -2^61)"] = (at(-B + 1, dim), at(1, dim), [], [[], [], []])
        L[f"{dn}: alloc 2^61-1, overhead -1 (sched 2^61)"] = (at(B - 1, dim), at(-1, dim), [], [[], [], []])
        L[f"{dn}: alloc 2^60, reservation -2^60 (avail 2^61)"] = (at(1 << 60, dim), None, *rows([-(1 << 60)], dim))
        L[f"{dn}: alloc 2^60, reservation -2^60+1 (avail 2^61-1)"] = (at(1 << 60, dim), None, *rows([-(1 << 60) + 1], dim))
        L[f"{dn}: overhead 2^60 twice under a zero reservation (first fit -2^61)"] = (at(0, dim), at(1 << 60, dim), *rows([0], dim))
        L[f"{dn}: overhead 2^60-1 twice under a zero reservation (first fit -2^61+2)"] = (at(0, dim), at((1 << 60) - 1, dim), *rows([0], dim))
        L[f"{dn}: alloc 2^61-1, overhead 2^61-1, reservation -2^61+1 (avail 2^61-1)"] = (at(B - 1, dim), at(B - 1, dim), *rows([-B + 1], dim))
        # sums of many small reservations
        L[f"{dn}: 1024 reservations of 2^51 (sum 2^61)"] = (at(0, dim), None, *rows([1 << 51] * 1024, dim))
        L[f"{dn}: 1023 reservations of 2^51 and one of 2^51-1 (sum 2^61-1)"] = (at(0, dim), None, *rows([1 << 51] * 1023 + [(1 << 51) - 1], dim))
        L[f"{dn}: sum 2^61 against alloc 1 (avail -2^61+1, sum outside)"] = (at(1, dim), None, *rows([1 << 51] * 1024, dim))
        # exact sums beyond 2^63 / 2^64 whose wrapped value looks harmless
        L[f"{dn}: 8 reservations of 2^60 (sum 2^63, wraps negative)"] = (at(0, dim), None, *rows([1 << 60] * 8, dim))
        L[f"{dn}: 16 reservations of 2^60 (sum 2^64, wraps to 0)"] = (at(0, dim), None, *rows([1 << 60] * 16, dim))
        L[f"{dn}: 16 reservations of 2^60 and one of 5 (wraps to 5)"] = (at(100, dim), None, *rows([1 << 60] * 16 + [5], dim))
        L[f"{dn}: 16 reservations of -2^60 (sum -2^64, wraps to 0)"] = (at(0, dim), None, *rows([-(1 << 60)] * 16, dim))
        L[f"{dn}: 4097 reservations of 2^52 (sum 2^64 + 2^52, wraps to 2^52)"] = (at(1 << 53, dim), None, *rows([1 << 52] * 4097, dim))
        # partial sums far outside, the exact sum small: representable, and must be exact
        L[f"{dn}: 8 of 2^60, 8 of -2^60 and 7 (sum 7)"] = (at(10, dim), None, *rows([1 << 60] * 8 + [-(1 << 60)] * 8 + [7], dim))
        L[f"{dn}: 300 of 2^61-1 and 300 of -2^61+1 (sum 0)"] = (at(10, dim), None, *rows([B - 1] * 300 + [-B + 1] * 300, dim))
    return L


LATTICE = _lattice()
# the points a 64-bit sum modulo 2^64 answers wrongly without an error, among those every input of which is in the domain
_MUST_REFUSE = ("(avail 2^61)", "(avail -2^61)", "(sched -2^61)", "(sched 2^61)", "(sum 2^61)", "sum outside", "wraps")


@pytest.fixture(scope="module")
def resident(packer):
    """a small valid snapshot and what a FIFO batch on a copy of it decides: what every refusal must leave in place"""
    rng = np.random.default_rng(17)
    n = 64
    alloc = (rng.integers(2, 17, n) * 1000, rng.integers(4, 65, n) << 30, np.zeros(n, I64))
    rnode = rng.integers(-1, n, 40).astype(I32)
    res = (rng.integers(0, 5, 40) * 500, rng.integers(0, 5, 40) << 29, np.zeros(40, I64))
    apps = dict(drv_cpu=[1000, 2000, 500, 4000], drv_mem=[1 << 30, 2 << 30, 1 << 29, 8 << 30], exe_cpu=[2000, 1000, 3000, 500],
                exe_mem=[4 << 30, 1 << 30, 2 << 30, 1 << 29], count=[3, 1, 5, 2])

    def prepare():
        packer.prepare_cluster(alloc, None, rnode, res)

    prepare()
    snap = [x.copy() for x in packer.get_snapshot()]
    want = packer.pack_batch(apps, 0, 0)
    return prepare, snap, apps, want


@pytest.mark.parametrize("point", list(LATTICE))
def test_domain_lattice(gangpack, packer, resident, point):
    prepare, snap, apps, want = resident
    prepare()
    alloc, over, rnode, res = LATTICE[point]
    refused = check_entries(gangpack, packer, alloc, over, rnode, res, point)
    if any(k in point for k in _MUST_REFUSE):
        assert len(refused) == 5, (point, refused)
    if {"gp_prepare_cluster", "gp_prepare_cluster_zones"} <= refused:
        # neither replaced the snapshot: the resident one is intact and packs as before
        for x, y in zip(packer.get_snapshot(), snap):
            assert np.array_equal(x, y), point
        got = packer.pack_batch(apps, 0, 0)
        for w, g in zip(want, got):
            assert np.array_equal(w, g), point


def test_refusal_message_and_recovery(gangpack, packer):
    z = np.zeros(2, I64)
    with pytest.raises(gangpack.native.GangpackError) as ei:
        packer.build_availability((np.array([B, 0]), z, z), None, np.zeros(0, I32), (z[:0], z[:0], z[:0]))
    assert ei.value.status == UNREPRESENTABLE and "gp_build_availability: " in str(ei.value) and "2^61" in str(ei.value)
    with pytest.raises(gangpack.native.GangpackError) as ei:
        packer.prepare_cluster((z, z, z), None, np.zeros(16, I32), (np.full(16, 1 << 60), np.zeros(16, I64), np.zeros(16, I64)))
    assert ei.value.status == UNREPRESENTABLE and "gp_prepare_cluster: " in str(ei.value) and "reservation sum" in str(ei.value)
    av, _ = packer.build_availability((np.array([B - 1, 0]), z, z), None, np.zeros(0, I32), (z[:0], z[:0], z[:0]))
    assert av[0].tolist() == [B - 1, 0]


# ---- zone totals: exact, whatever they add up to ---------------------------------------------------------------------------

@pytest.mark.parametrize("k", (4, 5, 8, 16, 4097))
@pytest.mark.parametrize("sign", (1, -1))
def test_zone_totals_beyond_64_bits(gangpack, packer, k, sign):
    """k nodes of +-(2^61 - 1) memory in zone 0 (from 5 on the total passes 2^63; 8 wraps to -8, 16 to -16 modulo 2^64), small
    nodes in zones 1 and 2: the order follows the exact totals through every entry that ranks zones"""
    big = sign * (B - 1)
    mem = np.array([big] * k + [7, 3, -5], I64)
    cpu = np.array([1000] * k + [1, 2, 3], I64)
    zid = np.array([0] * k + [1, 2, 2], I32)
    n = k + 3
    rank = np.random.default_rng(k).permutation(n).astype(I32)
    want = fr.priority_order(cpu.tolist(), mem.tolist(), zid.tolist(), 3, rank.tolist())
    assert (zid[want[0]] == 0) == (sign < 0)
    d, e = packer.potential_nodes(cpu, mem, zid, 3, rank)
    assert np.array_equal(d, want) and np.array_equal(e, want)
    rn, res = np.zeros(0, I32), (np.zeros(0, I64),) * 3
    out = packer.prepare_cluster_zones((cpu, mem, np.zeros(n, I64)), None, rn, res, zone_id=zid, n_zones=3, name_rank=rank)
    prio = fr.zone_priority(cpu.tolist(), mem.tolist(), zid.tolist(), 3)
    assert out["zone_of_group"][:3].tolist() == sorted(range(3), key=lambda z: prio[z])
    # first fit of a small request: the first node of the exact order it fits on
    em = 4 if sign > 0 else 0
    got, _ = packer.reschedule_from_reservations((cpu, mem, np.zeros(n, I64)), None, rn, res, (np.array([1], I64), np.array([em], I64)),
                                                 zone_id=zid, n_zones=3, name_rank=rank)
    assert got[0] == next(i for i in want if cpu[i] >= 1 and mem[i] >= em)
