"""The node priority orders of the snapshot front end (gp_zone_totals, gp_zone_priority, gp_make_keys, gp_sort_tiles,
gp_rank_by_search, gp_scatter_order, gp_split_candidates, the label re-sort) against frontend_ref's sorted() over Python
integers, at the sizes where the kernels change behaviour: the 4 096-key sort tile, the 8 192 positions a step of
gp_split_candidates covers, the 256 zones of one gp_zone_priority CTA, keys that differ in one 32-bit word or in sign only, and
candidate counts that cut the label re-sort's tiles while the node count cuts its grids.  Every order is asked of
gp_potential_nodes, of gp_prepare_cluster_zones (its undivided orders, or its per-zone groups) and, through first-fit decisions
over masks that drop a prefix of the order, of gp_reschedule_from_reservations, which ranks keys without sorting."""
import ctypes as C
import functools

import numpy as np
import pytest

import frontend_ref as fr
from k8s_spark_scheduler_b200 import native

pytestmark = pytest.mark.gpu

I64 = np.int64
EDGE = (1 << 61) - 1
SIZES = (1, 2, 31, 32, 33, 4095, 4096, 4097, 8191, 8192, 8193, 12288)
LARGE = (50000, 131073)


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def _draw(rng, values, n):
    return np.array(values, I64)[rng.integers(0, len(values), n)]


A = 5 * (1 << 32) + 7
WORDS = (A, A + 1, A + (1 << 32), A - (1 << 32))            # differ in the low word only, or in the high word only
KEY_CLASSES = {
    "equal": lambda rng, n: (np.full(n, 3000, I64), np.full(n, 8 << 30, I64)),
    "null_rank": lambda rng, n: (rng.integers(0, 6, n) * 1000, rng.integers(0, 5, n) * (1 << 30)),
    "mem_words": lambda rng, n: (np.full(n, 1000, I64), _draw(rng, WORDS, n)),
    "cpu_words": lambda rng, n: (_draw(rng, WORDS, n), np.full(n, 4 << 30, I64)),
    "negative": lambda rng, n: (-rng.integers(1, 6, n) * 1000, -rng.integers(1, 5, n) * (1 << 33)),
    "mixed_sign": lambda rng, n: (_draw(rng, (-(3 << 40), -1, 0, 1, 1 << 40), n), _draw(rng, (-(1 << 62) // 3, -(1 << 32), -1, 0, 1 << 32), n)),
    "edges": lambda rng, n: (_draw(rng, (-EDGE, -1, 0, 1, EDGE), n), _draw(rng, (-EDGE, -EDGE + 1, 0, EDGE - 1, EDGE), n)),
    "heavy": lambda rng, n: (rng.integers(0, 6, n) * 1000, rng.integers(0, 5, n) * (1 << 30)),
}


@functools.lru_cache(maxsize=None)
def cluster(cls, n, n_zones=1, zones="none"):
    """one seeded cluster: columns, masks, and frontend_ref's priority order of all its nodes"""
    rng = np.random.default_rng([sum(map(ord, cls)), n, n_zones, sum(map(ord, zones))])
    cpu, mem = (np.asarray(x, I64) for x in KEY_CLASSES[cls](rng, n))
    zid = None
    if zones == "spread":                                   # every id used (when n allows), sizes uneven
        zid = rng.integers(0, n_zones, n).astype(np.int32)
    elif zones == "gaps":                                   # every third id has no node
        zid = (rng.integers(0, max(n_zones // 3, 1), n) * 3 % n_zones).astype(np.int32)
    elif zones == "one_each":                               # n_zones == n, one node per zone
        zid = rng.permutation(n).astype(np.int32)
    c = dict(n=n, cpu=cpu, mem=mem, gpu=np.zeros(n, I64), zid=zid, nz=n_zones,
             rank=None if cls == "null_rank" else rng.permutation(n).astype(np.int32),
             cand=(rng.random(n) < 0.6).astype(np.uint8), unsched=(rng.random(n) < 0.1).astype(np.uint8),
             ready=(rng.random(n) < 0.9).astype(np.uint8), lr_d=None, lr_e=None)
    c["order"] = fr.priority_order(cpu.tolist(), mem.tolist(), None if zid is None else zid.tolist(), n_zones,
                                   None if c["rank"] is None else c["rank"].tolist())
    return c


def want_orders(c, **over):
    """frontend_ref's (driver order, executor order) of the cluster with some masks / label ranks replaced"""
    k = {**c, **over}
    drv = [i for i in c["order"] if k["cand"] is None or k["cand"][i]]
    exe = [i for i in c["order"] if not (k["unsched"] is not None and k["unsched"][i]) and (k["ready"] is None or k["ready"][i])]
    return fr.label_sort(drv, k["lr_d"]), fr.label_sort(exe, k["lr_e"])


def sort_args(c, **over):
    k = {**c, **over}
    return dict(zone_id=k["zid"], n_zones=k["nz"], name_rank=k["rank"], is_driver_candidate=k["cand"], unschedulable=k["unsched"],
                ready=k["ready"], driver_label_rank=k["lr_d"], executor_label_rank=k["lr_e"])


def no_res():
    return np.zeros(0, np.int32), (np.zeros(0, I64), np.zeros(0, I64), np.zeros(0, I64))


def check_potential_nodes(p, c, wd, we, **over):
    d, e = p.potential_nodes(c["cpu"], c["mem"], avail_gpu=c["gpu"], **sort_args(c, **over))
    assert np.array_equal(d, wd), "gp_potential_nodes: driver order"
    assert np.array_equal(e, we), "gp_potential_nodes: executor order"


def check_prepare_zones(p, c, wd, we, **over):
    """the same orders through gp_prepare_cluster_zones (no reservations: availability = allocatable).  One zone: the layout
    is the undivided orders.  Several: every candidate zone's group is the undivided order restricted to that zone, and the
    trailing group the rest of it."""
    rn, res = no_res()
    out = p.prepare_cluster_zones((c["cpu"], c["mem"], c["gpu"]), None, rn, res, **sort_args(c, **over))
    assert (out["n_driver"], out["n_executor"]) == (len(wd), len(we))
    snap = p.get_snapshot()
    assert np.array_equal(snap[0], c["cpu"]) and np.array_equal(snap[1], c["mem"])
    if c["zid"] is None or c["nz"] == 1:
        if len(wd) and len(we):
            assert out["n_zones"] == 1 and np.array_equal(out["drv_order"], wd) and np.array_equal(out["exec_order"], we)
        else:                                               # no candidate zone: everything in the trailing group
            assert out["n_zones"] == 0 and np.array_equal(out["drv_order"], wd) and np.array_equal(out["exec_order"], we)
        return
    zid, G = c["zid"], out["n_groups"]
    zog = out["zone_of_group"][:G]
    wd, we = np.asarray(wd, np.int32), np.asarray(we, np.int32)
    is_cand = np.zeros(c["nz"], bool)
    is_cand[zog[zog >= 0]] = True
    for g in range(G):
        for want, off, got in ((wd, out["drv_off"], out["drv_order"]), (we, out["exec_off"], out["exec_order"])):
            sel = want[zid[want] == zog[g]] if zog[g] >= 0 else want[~is_cand[zid[want]]]
            assert np.array_equal(got[off[g]:off[g + 1]], sel), ("group", g)


def check_first_fit(p, c, we):
    """gp_reschedule_from_reservations never sorts: with `unschedulable` dropping a prefix of the reference executor order,
    first fit must return the first remaining node of that order the request fits on"""
    if not len(we):
        return
    rn, res = no_res()
    exe = (np.array([0, 1000, 3000], I64), np.array([0, 1 << 30, A], I64))
    cpu, mem = c["cpu"].tolist(), c["mem"].tolist()
    for drop in sorted({0, 1, len(we) // 2, len(we) - 1}):
        unsched = np.array(c["unsched"], np.uint8)
        unsched[np.asarray(we[:drop], np.int64)] = 1
        got, _ = p.reschedule_from_reservations((c["cpu"], c["mem"], c["gpu"]), None, rn, res, exe, zone_id=c["zid"], n_zones=c["nz"],
                                                name_rank=c["rank"], unschedulable=unsched, ready=c["ready"],
                                                executor_label_rank=c["lr_e"])
        for x in range(3):
            ec, em = int(exe[0][x]), int(exe[1][x])
            want = next((i for i in we[drop:] if cpu[i] >= ec and mem[i] >= em), -1)
            assert got[x] == want, ("first fit", drop, x)


@pytest.mark.parametrize("n", SIZES + LARGE)
@pytest.mark.parametrize("cls", list(KEY_CLASSES))
def test_key_classes(packer, cls, n):
    if n in LARGE and cls not in ("heavy", "edges", "mem_words"):
        pytest.skip("the largest sizes run a selection of the key classes")
    c = cluster(cls, n)
    wd, we = want_orders(c)
    check_potential_nodes(packer, c, wd, we)
    check_prepare_zones(packer, c, wd, we)
    check_first_fit(packer, c, we)


ZONE_CASES = [(cls, n, nz, how) for cls in ("heavy", "mixed_sign") for n in (33, 4097, 12288)
              for nz, how in ((2, "spread"), (4, "spread"), (256, "spread"), (257, "spread"), (1000, "spread"), (257, "gaps"), (1000, "gaps"))]
ZONE_CASES += [("heavy", n, n, "one_each") for n in (257, 4097)] + [("equal", 4096, 8, "spread"), ("heavy", 50000, 257, "gaps"),
                                                                     ("edges", 8193, 4, "spread"), ("cpu_words", 4097, 256, "spread")]


@pytest.mark.parametrize("cls,n,nz,how", ZONE_CASES)
def test_zones(packer, cls, n, nz, how):
    """zone priorities from exact totals over every zone id: more zones than one gp_zone_priority CTA ranks, ids without a
    node ("gaps": each totals (0, 0), so they tie with one another and rank by id), negative totals and totals beyond 2^63
    (mixed_sign, edges), one node per zone."""
    c = cluster(cls, n, nz, how)
    wd, we = want_orders(c)
    check_potential_nodes(packer, c, wd, we)
    if how != "one_each":
        check_prepare_zones(packer, c, wd, we)
    check_first_fit(packer, c, we)


def test_tied_zone_totals_rank_by_id(packer):
    """equal (memory, cpu) totals: the library's documented choice is the zone id, also where only cpu differs"""
    n = 6 * 683                                                 # 4 098 nodes, 683 per zone
    zid = (np.arange(n) % 6).astype(np.int32)
    cpu = np.where(zid == 4, 999, 1000).astype(I64)             # zones 0-3, 5 tie; zone 4 is smaller in cpu alone
    mem = np.full(n, 1 << 30, I64)
    rank = np.random.default_rng(3).permutation(n).astype(np.int32)
    d, e = packer.potential_nodes(cpu, mem, zid, 6, rank)
    assert fr.zone_totals_tied(cpu.tolist(), mem.tolist(), zid.tolist(), 6)
    assert [int(zid[i]) for i in d[::n // 6]] == [4, 0, 1, 2, 3, 5]
    want = fr.priority_order(cpu.tolist(), mem.tolist(), zid.tolist(), 6, rank.tolist())
    assert np.array_equal(d, want) and np.array_equal(e, want)


LABELS = {
    "both": lambda rng, n: (rng.integers(-1, 4, n).astype(np.int32), rng.integers(-1, 3, n).astype(np.int32)),
    "all_unknown": lambda rng, n: (np.full(n, -1, np.int32), np.full(n, -1, np.int32)),
    "all_equal": lambda rng, n: (np.full(n, 2, np.int32), np.full(n, 0, np.int32)),
    "far_apart": lambda rng, n: (_draw(rng, (0, (1 << 31) - 2), n).astype(np.int32), _draw(rng, ((1 << 31) - 2, 0, -1), n).astype(np.int32)),
    "driver_only": lambda rng, n: (rng.integers(-1, 4, n).astype(np.int32), None),
    "executor_only": lambda rng, n: (None, rng.integers(-1, 4, n).astype(np.int32)),
}


@pytest.mark.parametrize("label", list(LABELS))
@pytest.mark.parametrize("count", (0, 1, 4095, 4096, 4097))
@pytest.mark.parametrize("n", (8193, 50000))
def test_candidate_counts_and_labels(packer, n, count, label):
    """`count` driver candidates (the nodes of lowest index) beside two thirds of the nodes as executor candidates, then the
    reverse: the re-sort's tiles are cut by the count on the device, its grids by n.  A count of 0 is an empty list and
    leaves the other list right."""
    c = cluster("heavy", n)
    lr_d, lr_e = LABELS[label](np.random.default_rng(n + count), n)
    idx = np.arange(n)
    few, many = (idx < count).astype(np.uint8), (idx % 3 != 0).astype(np.uint8)
    for cand, ready in ((few, many), (many, few)):
        over = dict(cand=cand, ready=ready, unsched=None, lr_d=lr_d, lr_e=lr_e)
        wd, we = want_orders(c, **over)
        assert count in (len(wd), len(we))
        check_potential_nodes(packer, c, wd, we, **over)
        if n == 8193:
            check_prepare_zones(packer, c, wd, we, **over)
    if count == 0:                                          # both lists empty
        over = dict(cand=few, ready=few, unsched=None, lr_d=lr_d, lr_e=lr_e)
        check_potential_nodes(packer, c, [], [], **over)


def _ties_through_every_entry(p, c, gpu):
    keys = fr.node_keys(c["cpu"].tolist(), c["mem"].tolist())
    want = fr.undefined_ties(c["order"], keys, gpu.tolist())
    args = sort_args(c)
    p.potential_nodes(c["cpu"], c["mem"], avail_gpu=gpu, **args)
    assert p.undefined_ties == want, "gp_potential_nodes"
    rn, res = no_res()
    # gp_prepare_cluster through the C ABI: the binding's prepare_cluster does not ask for the count
    ties = C.c_int32(-1)
    ui = native._usage_input((c["cpu"], c["mem"], gpu), None, rn, res)
    si = native._sort_input(c["n"], c["nz"], c["zid"], c["rank"], c["cand"], c["unsched"], c["ready"], ties=ties)
    assert native.load().gp_prepare_cluster(p._h, C.byref(ui), C.byref(si), None, None) == 0
    p.n_nodes = c["n"]
    assert ties.value == want, "gp_prepare_cluster"
    out = p.prepare_cluster_zones((c["cpu"], c["mem"], gpu), None, rn, res, layout=False, **args)
    assert out["undefined_ties"] == want, "gp_prepare_cluster_zones"
    return want


BOUNDARIES = (8, 256, 8192, 16384)                          # a thread's 8 positions, a warp's 256, a step's 8 192, the next step


@pytest.mark.parametrize("at", [(b,) for b in BOUNDARIES] + [BOUNDARIES])
def test_undefined_ties_at_the_split_boundaries(packer, at):
    """every key equal, so every adjacent pair ties on (zone priority, memory, cpu); gpu changes between positions b - 1 and
    b of the order, for the chosen b, and nowhere else"""
    c = cluster("equal", 20000)
    gpu = np.zeros(c["n"], I64)
    gpu[np.asarray(c["order"])] = np.searchsorted(np.array(at), np.arange(c["n"]), side="right")
    assert _ties_through_every_entry(packer, c, gpu) == len(at)


@pytest.mark.parametrize("n", (4097, 12288, 50000))
def test_undefined_ties_random_gpu(packer, n):
    c = cluster("heavy", n)
    gpu = np.random.default_rng(n).integers(0, 3, n).astype(I64)
    assert _ties_through_every_entry(packer, c, gpu) > n // 4


def test_scratch_reuse(gangpack, packer):
    """the main sort and both re-sorts share their scratch across calls of any size: a context that has just sorted the
    largest cluster answers smaller and differently shaped ones as a fresh context does"""
    rng = np.random.default_rng(9)
    seq = [(cluster("heavy", 131073), {}), (cluster("heavy", 1), {}),
           (cluster("heavy", 4097), dict(lr_d=rng.integers(-1, 3, 4097).astype(np.int32), lr_e=rng.integers(-1, 3, 4097).astype(np.int32))),
           (cluster("heavy", 4097, 257, "gaps"), {}), (cluster("heavy", 33, 4, "spread"), {})]
    used = gangpack.GangPacker()
    try:
        for c, over in seq:
            wd, we = want_orders(c, **over)
            check_potential_nodes(used, c, wd, we, **over)
            check_prepare_zones(used, c, wd, we, **over)
            fresh = gangpack.GangPacker()
            try:
                check_potential_nodes(fresh, c, wd, we, **over)
            finally:
                fresh.close()
    finally:
        used.close()
