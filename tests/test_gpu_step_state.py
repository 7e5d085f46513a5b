"""State a call leaves on its context for the next one: the snapshot layout and the independent tables path zero or
rewrite every word they rely on themselves (node_slot, drv_pos, SnapMeta, the table set's counters, hash keys and
look-back words, the status block), with no memset between calls.  One long-lived context runs a sequence of layouts
and pack calls that change every size those words depend on; after each call it must return what a fresh context
returns for the same call (placements, statistics, status), and a captured snapshot + pack graph must replay the same."""
import os

import numpy as np
import pytest

from helpers import random_apps, random_cluster

pytestmark = pytest.mark.gpu
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group")
STATS = ("nodes_scanned", "drivers_tried", "scan_path_apps", "scan_path_nodes")


def layout(rng, n, n_groups):
    """Every node is in one group or in none; in its group it is an executor and driver candidate, an executor candidate
    only, or a driver candidate only.  Some groups are empty."""
    cpu, mem, gpu = random_cluster(rng, n, negative=bool(rng.integers(0, 2)), gpus=True)
    grp = rng.integers(-1, n_groups, n)
    if n_groups > 2:
        grp[grp == 1] = -1                                    # group 1 stays empty
    role = rng.choice(3, n, p=[0.7, 0.15, 0.15])             # 0 both, 1 executor only, 2 driver only
    eorder, dorder, eoff, doff = [], [], [0], [0]
    for g in range(n_groups):
        e = rng.permutation(np.nonzero((grp == g) & (role != 2))[0])
        d = rng.permutation(np.nonzero((grp == g) & (role != 1))[0])
        eorder.append(e); dorder.append(d)
        eoff.append(eoff[-1] + len(e)); doff.append(doff[-1] + len(d))
    cat = lambda xs: np.concatenate(xs).astype(np.int32)
    return cpu, mem, gpu, cat(eorder), cat(dorder), np.array(eoff, np.int32), np.array(doff, np.int32)


def apps_for(rng, q, n_groups, shapes=6):
    """At most 64 executor and driver shapes, every one with its tables, make the statistics a function of the inputs;
    with more, which shapes get tables depends on the order the threads claim them, so only the placements are."""
    a = random_apps(rng, q, gpus=True, big_counts=True)
    k = rng.integers(0, shapes, q)
    a["exe_cpu"] = (k * 10 + 100).astype(np.int64)
    a["exe_mem"] = ((k % 7 + 1) << 28).astype(np.int64)
    a["exe_gpu"] = (k % 2).astype(np.int64)
    a["group"] = rng.integers(0, n_groups, q).astype(np.int32)
    return a


def fitted(dn, en, off):
    """ExecutorNodes with the slices of applications that did not fit set to -1 (their contents are unspecified)"""
    en = np.asarray(en).astype(np.int64).copy()
    for i in np.nonzero(np.asarray(dn) < 0)[0]:
        en[off[i]:off[i + 1]] = -1
    return en[:int(off[-1])]


def outcome(fn):
    try:
        return ("ok", fn())
    except Exception as e:                                    # GangpackError: compare the status, not the text
        return ("err", getattr(e, "status", type(e).__name__))


def host_calls(p, snap, ops):
    """gp_set_snapshot, then each op; every result copied out."""
    out = [outcome(lambda: p.set_snapshot(*snap))]
    for op in ops:
        out.append(outcome(lambda: op(p)))
    return out


def pack(a, algo, mode=0, wire=None, stats=True):
    def run(p):
        dn, en, off = p.pack_batch(a, algo, mode, wire=wire)
        st = p.stats()
        return dn.copy(), fitted(dn, en, off), off.copy(), [st[k] for k in STATS] if stats else None
    return run


def after_pack(a, algo):
    """a pack, then the reservation-driven calls on its placements and the snapshot they leave"""
    def run(p):
        dn, en, off = p.pack_batch(a, algo, 0)
        placed = (dn.copy(), fitted(dn, en, off).astype(np.int32), off.copy())
        cpu, mem, gpu = p.get_snapshot()
        p.set_schedulable(cpu.clip(0) + 1000, mem.clip(0) + (1 << 30), gpu.clip(0) + 1)
        eff = p.packing_efficiency(a, placed, algo)
        rows = p.reserve_placements(a, placed, subtract=True)
        return placed, eff, {k: np.asarray(v).copy() for k, v in rows.items()}, p.get_snapshot()
    return run


def zones(z, snap):
    """single-az-tightly-pack over the snapshot's groups (it takes the independent tables path per zone)"""
    def run(p):
        p.set_schedulable(*[x.clip(0) for x in snap[:3]])
        out = [np.asarray(x).copy() for x in p.pack_batch_zones(z, 0)]
        out[2] = fitted(out[1], out[2], out[3])
        st = p.stats()
        return out, [st[k] for k in STATS]
    return run


def assert_same(got, want, label):
    assert type(got) is type(want), label
    if isinstance(got, dict):
        assert got.keys() == want.keys(), label
        for k in got:
            assert_same(got[k], want[k], f"{label}.{k}")
    elif isinstance(got, (tuple, list)):
        assert len(got) == len(want), label
        for i, (x, y) in enumerate(zip(got, want)):
            assert_same(x, y, f"{label}[{i}]")
    elif isinstance(got, np.ndarray):
        assert np.array_equal(got, want, equal_nan=got.dtype.kind == "f"), label
    else:
        assert got == want, label


def check_against_fresh(gangpack, long_lived, snap, ops, label):
    got = host_calls(long_lived, snap, ops)
    p = gangpack.GangPacker()
    try:
        want = host_calls(p, snap, ops)
    finally:
        p.close()
    assert_same(got, want, label)


def test_layouts_and_pack_calls_on_one_context(gangpack):
    rng = np.random.default_rng(2024)
    p = gangpack.GangPacker()
    tables_off = None
    try:
        # node table sizes and group counts that shrink, grow (reallocating every array) and shrink again
        for step, (n, n_groups) in enumerate([(3000, 3), (400, 1), (9000, 5), (9000, 2), (1200, 4), (20000, 3), (700, 6)]):
            snap = layout(rng, n, n_groups)
            a = apps_for(rng, 3000, n_groups)
            small = apps_for(rng, 20, n_groups)
            many = apps_for(rng, 2000, n_groups, shapes=150)
            bad = apps_for(rng, 500, n_groups)
            bad["count"][137] = -1
            ops = [
                pack(a, 0), pack(a, 1),
                pack(a, 0, wire=dict(quantity_bits=64, node_bits=16, offsets=False)),
                pack(a, 1, wire=dict(quantity_bits=64, node_bits=32, offsets=False)),
                pack(small, 0), pack(small, 1, wire=dict(quantity_bits=64, node_bits=32, offsets=False)),
                pack(many, 0, stats=False), pack(many, 1, stats=False),
                pack(bad, 0), pack(a, 0),
                pack(a, 0, mode=1), pack(a, 1),
                after_pack(a, 0),
            ]
            check_against_fresh(gangpack, p, snap, ops, f"layout {step}")
            # a GANGPACK_TABLES=0 context on the same calls, also never reset
            if tables_off is None:
                os.environ["GANGPACK_TABLES"] = "0"
                try:
                    tables_off = gangpack.GangPacker()
                finally:
                    os.environ.pop("GANGPACK_TABLES")
            got = host_calls(tables_off, snap, ops[:10])
            want = host_calls(p, snap, ops[:10])
            for i in (1, 2, 3, 4, 5, 6, 7, 8, 9, 10):     # placements agree; the statistics count different paths
                assert got[i][0] == want[i][0], (step, i)
                if got[i][0] == "ok":
                    assert_same(got[i][1][:3], want[i][1][:3], f"tables off, layout {step} op {i}")
    finally:
        p.close()
        if tables_off is not None:
            tables_off.close()


def test_multi_chunk_and_zone_calls_in_between(gangpack):
    rng = np.random.default_rng(77)
    os.environ["GANGPACK_CHUNK_APPS"] = "2048"
    try:
        p = gangpack.GangPacker()
    finally:
        os.environ.pop("GANGPACK_CHUNK_APPS")
    try:
        for step in range(3):
            n_groups = 3
            snap = layout(rng, 5000, n_groups)
            a = apps_for(rng, 9000, n_groups)
            z = apps_for(rng, 300, 1)
            z.pop("group")
            ops = [pack(a, 0), pack(a, 1, mode=2), pack(a, 1), zones(z, snap), pack(a, 0)]
            check_against_fresh(gangpack, p, snap, ops, f"chunked step {step}")
    finally:
        p.close()


def test_device_step_eager_and_graph_replay(gangpack):
    """gp_set_snapshot_device + gp_pack_batch_device (the call whose first classify tile zeroes the status block) on one
    context across layouts, against a fresh context; then the step captured into a CUDA graph and replayed 20 times."""
    import torch
    rng = np.random.default_rng(5)
    dev = torch.device("cuda", 0)
    t = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(dt).to(dev)

    def device_inputs(snap, a, offsets):
        cpu, mem, gpu, eo, do, eoff, doff = snap
        tn = (t(cpu, torch.int64), t(mem, torch.int64), t(gpu, torch.int64), t(eoff, torch.int32), t(eo, torch.int32),
              t(doff, torch.int32), t(do, torch.int32))
        ta = {k: t(a[k], torch.int64 if a[k].dtype == np.int64 else torch.int32) for k in KEYS}
        off = np.concatenate([[0], np.cumsum(a["count"].clip(0))]).astype(np.int64)
        if offsets:
            ta["off"] = t(off, torch.int64)
        d = torch.empty(len(a["count"]), dtype=torch.int32, device=dev)
        e = torch.empty(max(int(off[-1]), 1), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()                              # the library's stream does not wait for torch's
        return tn, ta, off, d, e

    def step(p, tn, ta, algo, d, e):
        p.set_snapshot_device(*tn)
        p.pack_batch_device(ta, algo, 0, d, e)

    def result(p, off, d, e):
        st = outcome(lambda: p.stats())                       # synchronises the library's stream
        if st[0] == "ok":
            st = ("ok", [st[1][k] for k in STATS])
        dn = d.cpu().numpy()
        return dn, fitted(dn, e.cpu().numpy(), off), st

    p = gangpack.GangPacker()
    try:
        for i, (n, g, q, algo, offsets) in enumerate([(3000, 3, 4000, 0, True), (500, 1, 20, 1, False), (9000, 4, 6000, 1, True),
                                                      (9000, 4, 6000, 0, False), (800, 2, 20, 0, True), (4000, 5, 3000, 0, True)]):
            snap = layout(rng, n, g)
            a = apps_for(rng, q, g)
            if i == 3:
                a["count"][5] = -2                            # a device-side validation error, then valid calls again
            tn, ta, off, d, e = device_inputs(snap, a, offsets)
            step(p, tn, ta, algo, d, e)
            got = result(p, off, d, e)
            f = gangpack.GangPacker()
            try:
                d2, e2 = torch.empty_like(d), torch.empty_like(e)
                step(f, tn, ta, algo, d2, e2)
                want = result(f, off, d2, e2)
            finally:
                f.close()
            assert_same(got, want, f"device step {i}")

        snap = layout(rng, 6000, 3)
        a = apps_for(rng, 5000, 3)
        tn, ta, off, d, e = device_inputs(snap, a, True)
        stream = torch.cuda.ExternalStream(p.stream_handle(), device=dev)
        with torch.cuda.stream(stream):
            for _ in range(3):
                step(p, tn, ta, 0, d, e)
            eager = result(p, off, d, e)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                step(p, tn, ta, 0, d, e)
            for r in range(20):
                d.fill_(-7); e.fill_(-7)
                graph.replay()
                stream.synchronize()
                assert_same(result(p, off, d, e), eager, f"replay {r}")
    finally:
        p.close()
