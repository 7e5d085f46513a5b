"""Shape interning of gp_decide_tables on crafted fingerprints, and 16-bit node indices above 2^15.

The classify phase interns executor and driver requests by their 64-bit fingerprint alone; decide_load then compares the
full tuple, so a colliding executor shape must go to the scan and a colliding driver shape must start its driver loop at 0.
The batches here are built from tests/fingerprint_ref.py (whose premises test_fingerprint_model.py checks): requests whose
fingerprints collide in all 64 bits, 17 requests sharing one home slot (a full 16-probe window that wraps past slot 1023),
and 64 / 65 / 300 distinct shapes around kMaxShapes.  A colliding request asks for 2^50 or more in its solved dimension,
so it fits no node and a mix-up in either direction changes a placement.  Every case is checked against the closed-form
oracle, the literal oracle and a GANGPACK_TABLES=0 context (every decision by the node-order scan), on a roomy cluster
where nothing else sends an application to the scan, so scan_path_apps shows whether the premise was met on the device."""
import itertools

import numpy as np
import pytest

import fingerprint_ref as fr
from helpers import assert_same_results, literal_batch, res_aos
from test_gpu_one_launch_decide import make_packer

pytestmark = pytest.mark.gpu
GI = 1 << 30
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")
DRIVER = (500, GI, 0)
EXEC = (1000, 4 * GI, 0)
N_SMALL = 600                 # driver candidates at the front of the driver order that no driver of these batches fits on


@pytest.fixture(scope="module")
def packers(gangpack):
    ps = (make_packer(gangpack), make_packer(gangpack, GANGPACK_TABLES=0))
    yield ps
    for p in ps:
        p.close()


def roomy_cluster(n=3000, seed=5):
    """Every executor request of the batches fits on most nodes many times over; the driver order starts with N_SMALL
    nodes of 400 millicores, so a driver's first fitting candidate lies deep in it."""
    rng = np.random.default_rng(seed)
    cpu = rng.integers(32, 65, n) * 1000
    mem = rng.integers(64, 257, n) * GI
    gpu = rng.integers(0, 9, n)
    small = rng.permutation(n)[:N_SMALL]
    cpu[small] = 400
    eorder = rng.permutation(n).astype(np.int32)
    rest = np.setdiff1d(np.arange(n), small)
    dorder = np.concatenate([small, rng.permutation(rest)]).astype(np.int32)
    return cpu.astype(np.int64), mem.astype(np.int64), gpu.astype(np.int64), eorder, dorder


CLUSTER = roomy_cluster()


def batch(drivers, executors, counts):
    """apps from per-application driver and executor tuples"""
    d, e = np.asarray(drivers, np.int64), np.asarray(executors, np.int64)
    return {"drv_cpu": d[:, 0].copy(), "drv_mem": d[:, 1].copy(), "drv_gpu": d[:, 2].copy(),
            "exe_cpu": e[:, 0].copy(), "exe_mem": e[:, 1].copy(), "exe_gpu": e[:, 2].copy(),
            "count": np.asarray(counts, np.int32)}


def run_checked(packers, oracle, a, algo, literal=True):
    """tables against the scan context, the closed-form oracle and (small batches) the literal oracle -> (results, stats)"""
    cpu, mem, gpu, eorder, dorder = CLUSTER
    got = []
    for p in packers:
        p.set_snapshot(cpu, mem, gpu, eorder, dorder)
        dn, en, off = p.pack_batch(a, algo, 0)
        got.append(((dn.copy(), np.asarray(en).astype(np.int32), off), p.stats()))
    (res, st), (scan, _) = got
    assert_same_results(res, scan, f"tables vs scan algo {algo}")
    drv, exe = res_aos(a["drv_cpu"], a["drv_mem"], a["drv_gpu"]), res_aos(a["exe_cpu"], a["exe_mem"], a["exe_gpu"])
    _, wd, we, woff, _ = oracle.closed_batch(algo, 0, cpu, mem, gpu, dorder, eorder, drv, exe, a["count"], None)
    assert_same_results(res, (wd, we, woff), f"closed oracle algo {algo}")
    if literal:
        assert_same_results(res, literal_batch(oracle, algo, cpu, mem, gpu, dorder, eorder, a), f"literal oracle algo {algo}")
    return res, st


# ---- the crafted batches ------------------------------------------------------------------------------------------------
COUNTS = [0, 0, 1, 1, 3, 2, 5, 4, 1, 0, 2]


def one_warp_executor_pairs(y_first):
    """q = 32, one warp: lane l carries pair l % 3, X and Y alternating from the pair's lowest lane (Y there when
    y_first).  -> (apps, number of applications whose tuple is not their pair's claimer's)"""
    pairs = fr.executor_pairs()
    exe, counts, losers = [], [], 0
    for lane in range(32):
        x, y = pairs[lane % 3]
        j = lane // 3
        is_y = (j % 2 == 0) == y_first
        exe.append(y if is_y else x)
        counts.append(COUNTS[j])
        losers += j % 2 == 1                       # the claimer is the pair's lane j = 0
    return batch([DRIVER] * 32, exe, counts), losers


def interleaved_executor_pairs(q=8192, seed=1):
    """pairs interleaved every few applications over 32 classify tiles -> (apps, possible scan_path_apps values)"""
    rng = np.random.default_rng(seed)
    pairs = fr.executor_pairs()
    which = rng.integers(0, 3, q)
    is_y = rng.random(q) < 0.5
    exe = [pairs[w][int(y)] for w, y in zip(which, is_y)]
    n = [(int(((which == p) & ~is_y).sum()), int(((which == p) & is_y).sum())) for p in range(3)]
    sums = {sum(c) for c in itertools.product(*n)}
    return batch([DRIVER] * q, exe, rng.integers(0, 6, q)), sums


def driver_pairs(y_first, q=64):
    x, y = fr.driver_pair()
    drivers = [(y if (lane % 2 == 0) == y_first else x) for lane in range(q)]
    return batch(drivers, [EXEC] * q, [COUNTS[i % len(COUNTS)] for i in range(q)])


def per_shape(shapes, per, seed, drivers=False):
    """`per` applications of each shape, shuffled, counts 0..5"""
    rng = np.random.default_rng(seed)
    idx = rng.permutation(np.repeat(np.arange(len(shapes)), per))
    tup = [shapes[i] for i in idx]
    counts = rng.integers(0, 6, len(idx))
    return batch(tup, [EXEC] * len(idx), counts) if drivers else batch([DRIVER] * len(idx), tup, counts)


def crafted_batches():
    """name -> (apps, allowed scan_path_apps values)"""
    out = {}
    for y_first in (False, True):
        a, losers = one_warp_executor_pairs(y_first)
        out[f"warp-exec-{'YX' if y_first else 'XY'}"] = (a, {losers})
        out[f"warp-drv-{'YX' if y_first else 'XY'}"] = (driver_pairs(y_first), {0})
    out["tiles-exec"] = interleaved_executor_pairs()
    ex, dr, mixed = fr.full_window_sets()
    out["window-exec"] = (per_shape(ex, 40, 1), {40})
    out["window-drv"] = (per_shape(dr, 40, 2, drivers=True), {0})
    out["window-mixed"] = (per_shape(mixed, 40, 3), {0, 40})
    sets = fr.shape_count_sets()
    out["exec64"] = (per_shape(sets["exec64"], 20, 4), {0})
    out["exec65"] = (per_shape(sets["exec65"], 20, 5), {20})
    for k in ("drv64", "drv65", "drv300"):
        out[k] = (per_shape(sets[k], 8, 6, drivers=True), {0})
    return out


BATCHES = crafted_batches()


@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("name", list(BATCHES))
def test_crafted_batch(oracle, packers, name, algo):
    a, allowed = BATCHES[name]
    res, st = run_checked(packers, oracle, a, algo, literal=len(a["count"]) <= 4096)
    assert st["scan_path_apps"] in allowed, (name, st["scan_path_apps"], allowed)
    dn = res[0]
    huge = (np.stack([a[k] for k in KEYS[:6]]) >= fr.HUGE).any(0)
    # the premise of a mix-up test: the colliding requests fit nowhere (count > 0), their partners do
    if huge.any():
        assert (dn[huge & (a["count"] > 0)] < 0).all()
        assert (dn[~huge] >= 0).all()


# ---- the other callers of the launch ------------------------------------------------------------------------------------
def test_device_entry_with_early_start(gangpack, packers):
    """The bench's form of the step: an async-snapshot context running set_snapshot_device + pack_batch_device, whose
    gp_decide_tables starts while the layout runs; eagerly and captured once into a CUDA graph and replayed."""
    import torch
    dev = torch.device("cuda", 0)
    cpu, mem, gpu, eorder, dorder = CLUSTER
    n = len(cpu)
    t = lambda v, dt: torch.from_numpy(np.ascontiguousarray(v, dt)).to(dev)
    snap = [t(cpu, np.int64), t(mem, np.int64), t(gpu, np.int64), t([0, n], np.int32), t(eorder, np.int32),
            t([0, n], np.int32), t(dorder, np.int32)]
    p = gangpack.GangPacker(async_snapshot=True)
    try:
        stream = torch.cuda.ExternalStream(p.stream_handle(), device=dev)
        for name, (a, allowed) in BATCHES.items():
            for algo in (0, 1):
                packers[1].set_snapshot(cpu, mem, gpu, eorder, dorder)
                want = packers[1].pack_batch(a, algo, 0)
                off = want[2]
                ta = {k: t(a[k], np.int32 if k == "count" else np.int64) for k in KEYS}
                ta["off"] = t(off, np.int64)
                d = torch.full((len(a["count"]),), -7, dtype=torch.int32, device=dev)
                e = torch.full((max(int(off[-1]), 1),), -7, dtype=torch.int32, device=dev)
                torch.cuda.synchronize()

                def step():
                    p.set_snapshot_device(*snap)
                    p.pack_batch_device(ta, algo, 0, d, e)

                step()
                assert p.stats()["scan_path_apps"] in allowed, (name, algo)
                assert_same_results((d.cpu().numpy(), e.cpu().numpy(), off), want, f"{name} eager algo {algo}")
                with torch.cuda.stream(stream):
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=stream):
                        step()
                    d.fill_(-7); e.fill_(-7)
                    graph.replay()
                p.synchronize()
                assert_same_results((d.cpu().numpy(), e.cpu().numpy(), off), want, f"{name} replay algo {algo}")
                del graph
    finally:
        p.close()


def test_zone_entry_points(packers):
    """gp_pack_batch_zones and gp_pack_batch_az_aware run the same launch: tables and scan give the same bits"""
    cpu, mem, gpu, _, dorder = CLUSTER
    n, Z = len(cpu), 3
    zone_of = np.arange(n) % (Z + 1)                 # zone Z: the trailing group of the az-aware layout
    eo = np.concatenate([dorder[zone_of[dorder] == z] for z in range(Z + 1)]).astype(np.int32)     # both orders: dorder
    eoff = np.array([0] + [int((zone_of == z).sum()) for z in range(Z + 1)], np.int32).cumsum().astype(np.int32)
    for name, (a, _) in BATCHES.items():
        outs = []
        for p in packers:
            p.set_snapshot(cpu, mem, gpu, eo[:eoff[Z]], eo[:eoff[Z]], eoff[:Z + 1], eoff[:Z + 1])
            p.set_schedulable(cpu, mem, gpu)
            z1 = [x.copy() for x in p.pack_batch_zones(a, 0)]
            p.set_snapshot(cpu, mem, gpu, eo, eo, eoff, eoff)
            p.set_schedulable(cpu, mem, gpu)
            z2 = [x.copy() for x in p.pack_batch_az_aware(a, dorder, dorder, Z)]
            outs.append((z1, z2))
        for x, y in zip(*outs):             # (zone, driver_node, executor_nodes, off, avg_efficiency) of each entry point
            assert np.array_equal(x[0], y[0]) and np.array_equal(x[4], y[4]), name
            assert_same_results(x[1:4], y[1:4], name)      # executor slices of unplaced applications are unspecified


# ---- 16-bit node indices ------------------------------------------------------------------------------------------------
N16 = 65535


def high_index_case(n=N16, q=20000):
    """synthetic nodes whose priority order starts at the highest indices; synthetic apps plus counts of 100-300, so the
    index-shift emission (k - 1 + delta < 256) and the table walk both write indices near 65 534"""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(n)
    order = np.arange(n - 1, -1, -1, dtype=np.int32)
    apps = synth.make_apps(q)
    a = {k: apps[k] for k in KEYS}
    rng = np.random.default_rng(16)
    big = rng.random(q) < 0.05
    a["count"] = np.where(big, rng.integers(100, 301, q), a["count"]).astype(np.int32)
    return nodes, order, a


@pytest.fixture(scope="module")
def case16():
    return high_index_case()


def wide(got):
    return got[0], np.asarray(got[1]).astype(np.int32), got[2]


@pytest.mark.parametrize("algo", [0, 1])
def test_sixteen_bit_indices_above_2_15(gangpack, oracle, case16, algo):
    nodes, order, a = case16
    q = len(a["count"])
    snap = (nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    p = gangpack.GangPacker()
    chunked = make_packer(gangpack, GANGPACK_CHUNK_APPS=4096)
    try:
        for x in (p, chunked):
            x.set_snapshot(*snap)
        want = wide(p.pack_batch(a, algo, 0))
        dn, en, off = want
        placed = np.concatenate([en[off[i]:off[i + 1]] for i in np.nonzero(dn >= 0)[0]])
        assert placed.max() > 65000 and (dn > 65000).any()
        assert (placed >= 1 << 15).mean() > 0.5
        w16 = dict(quantity_bits=64, node_bits=16)
        # pageable
        assert_same_results(wide(p.pack_batch(a, algo, 0, wire=dict(w16, offsets=False))), want, "pageable")
        # pinned inputs and pinned uint16 results
        pin = p.pinned_columns(q, [k for k in KEYS if k != "count"], dtype=np.int64)
        for k in pin:
            pin[k][:] = a[k]
        pin["count"] = p.pinned(q, np.int32); pin["count"][:] = a["count"]
        od, oe = p.pinned(q, np.int32), p.pinned(int(off[-1]), np.uint16)
        od[:] = -7; oe[:] = 7
        assert_same_results(wide(p.pack_batch(pin, algo, 0, out=(od, oe), wire=w16)), want, "pinned")
        # a pipelined batch of five chunks
        od[:] = -7; oe[:] = 7
        assert_same_results(wide(chunked.pack_batch(pin, algo, 0, out=(od, oe), wire=w16)), want, "chunked pinned")
        assert_same_results(wide(chunked.pack_batch(a, algo, 0, wire=w16)), want, "chunked pageable")
        # a sample against the oracle, big counts included
        rng = np.random.default_rng(algo)
        sel = np.concatenate([rng.choice(np.nonzero(a["count"] >= 100)[0], 40, replace=False),
                              rng.choice(np.nonzero(a["count"] < 100)[0], 60, replace=False)])
        sub = {k: a[k][sel] for k in KEYS}
        _, wd, we, woff, _ = oracle.closed_batch(algo, 0, *snap[:3], order, order, res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"]),
                                                 res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"]), sub["count"], None)
        got16 = wide(p.pack_batch(sub, algo, 0, wire=w16))
        assert_same_results(got16, (wd, we, woff), "sample vs oracle")
        assert got16[1].max() > 65000
    finally:
        p.close(); chunked.close()


def test_sixteen_bit_multi_context(gangpack, case16):
    nodes, order, a = case16
    snap = (nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    p = gangpack.GangPacker()
    m = gangpack.MultiGangPacker([0, 0, 0])
    try:
        p.set_snapshot(*snap)
        m.set_snapshot(*snap)
        for algo in (0, 1):
            want = wide(p.pack_batch(a, algo, 0))
            got = wide(m.pack_batch(a, algo, 0, wire=dict(quantity_bits=64, node_bits=16, offsets=False)))
            assert_same_results(got, want, f"multi algo {algo}")
            assert got[1].max() > 65000
    finally:
        m.close(); p.close()


def test_sixteen_bit_node_limit(gangpack):
    """65 536 nodes are refused with 16-bit indices (GP_ERR_INVALID), and the 32-bit layout takes them; 65 535 are accepted
    (test_sixteen_bit_indices_above_2_15)"""
    nodes, order, a = high_index_case(65536, 2000)
    p = gangpack.GangPacker()
    try:
        p.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
        with pytest.raises(gangpack.native.GangpackError, match="65535") as e:
            p.pack_batch(a, 0, 0, wire=dict(quantity_bits=64, node_bits=16))
        assert e.value.status == 1
        dn, en, _ = p.pack_batch(a, 0, 0, wire=dict(quantity_bits=64, node_bits=32))
        assert en.max() > 65000 and (dn >= 0).any()
    finally:
        p.close()
