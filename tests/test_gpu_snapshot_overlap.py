"""With GP_CFG_ASYNC_SNAPSHOT, a gp_pack_batch_device that directly follows gp_set_snapshot_device on the same stream
starts its gp_decide_tables while the slot layout still runs: its classify tiles read only the application columns, and
everything that reads the snapshot (the segment prefix, the groups, the maxima behind the division classes) waits for
the layout.  These tests change the snapshot between steps so that a read placed before that wait would see the
previous step's layout, and compare every step with a context without the flag on the same inputs."""
import numpy as np
import pytest

from helpers import random_apps, random_cluster

pytestmark = pytest.mark.gpu
KEYS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group", "off")
STATS = ("nodes_scanned", "drivers_tried", "scan_path_apps", "scan_path_nodes")
N, G, Q = 6000, 4, 5000
# executor-order length of each group; every boundary of a 1024-node table segment is crossed one way or the other,
# and one group is empty
SIZES = [(1024, 1025, 2047, 1904), (1023, 3073, 1, 1903), (0, 4097, 1000, 903), (2048, 2048, 1024, 880)]


def snapshot(rng, sizes, kind):
    """kind 0: ordinary values; 1: cpu and memory availability above 2^32 (other compact-view shifts, other arithmetic
    classes); 2: negative GPU availability"""
    cpu, mem, gpu = random_cluster(rng, N, gpus=True, negative=kind == 2)
    if kind == 1:
        big = rng.integers(0, 4, N) == 0
        cpu = np.where(big, rng.integers(1, 1 << 12, N) << 33, cpu)
        mem = np.where(big, rng.integers(1, 1 << 8, N) << 41, mem)
    if kind == 2:
        gpu = np.where(rng.integers(0, 6, N) == 0, -1, gpu)
    perm = rng.permutation(N)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    dorder = np.concatenate([rng.permutation(perm[off[g]:off[g + 1]]) for g in range(G)])
    return {"cpu": cpu.astype(np.int64), "mem": mem.astype(np.int64), "gpu": gpu.astype(np.int64), "eoff": off,
            "eorder": perm.astype(np.int32), "doff": off, "dorder": dorder.astype(np.int32)}


def apps(rng):
    """At most 64 executor and driver shapes: the statistics are then a function of the inputs too"""
    a = random_apps(rng, Q, gpus=True, big_counts=True)
    k = rng.integers(0, 8, Q)
    a["exe_cpu"] = (k * 250 + 250).astype(np.int64)
    a["exe_mem"] = ((k % 5 + 1) << 28).astype(np.int64) + (k == 3) * 7
    a["exe_gpu"] = (k % 2).astype(np.int64)
    a["group"] = rng.integers(0, G, Q).astype(np.int32)
    a["off"] = np.concatenate([[0], np.cumsum(a["count"].clip(0))]).astype(np.int64)
    return a


def fitted(dn, en, off):
    en = en.astype(np.int64).copy()
    for i in np.nonzero(dn < 0)[0]:
        en[off[i]:off[i + 1]] = -1
    return en[:int(off[-1])]


class Step:
    """Device tensors of one snapshot-and-pack step, sized once; put() rewrites their contents on `stream` from device
    copies of a case made beforehand (no allocation on the library's stream, which dies with its context)."""

    def __init__(self, torch, dev, exec_cap):
        self.torch, self.dev = torch, dev
        z = lambda n, dt: torch.zeros(n, dtype=dt, device=dev)
        self.tn = {"cpu": z(N, torch.int64), "mem": z(N, torch.int64), "gpu": z(N, torch.int64), "eoff": z(G + 1, torch.int32),
                   "eorder": z(N, torch.int32), "doff": z(G + 1, torch.int32), "dorder": z(N, torch.int32)}
        self.ta = {k: z(Q + (k == "off"), torch.int64 if k not in ("count", "group") else torch.int32) for k in KEYS}
        self.d = z(Q, torch.int32)
        self.e = z(exec_cap, torch.int32)

    def upload(self, snap, a):
        t = lambda v: self.torch.from_numpy(np.ascontiguousarray(v)).to(self.dev)
        return {k: t(v) for k, v in snap.items()}, {k: t(a[k]) for k in KEYS}

    def put(self, dev_case, stream):
        with self.torch.cuda.stream(stream):
            for k, v in dev_case[0].items():
                self.tn[k].copy_(v)
            for k, v in dev_case[1].items():
                self.ta[k].copy_(v)

    def snapshot(self, p, stream=0):
        t = self.tn
        p.set_snapshot_device(t["cpu"], t["mem"], t["gpu"], t["eoff"], t["eorder"], t["doff"], t["dorder"], stream=stream)

    def pack(self, p, algo, stream=0):
        p.pack_batch_device(self.ta, algo, 0, self.d, self.e, stream=stream)

    def result(self, p, a):
        st = p.stats()                                       # synchronises the context's stream
        dn = self.d.cpu().numpy()
        return dn, fitted(dn, self.e.cpu().numpy(), a["off"]), [st[k] for k in STATS]


def reference(gangpack, torch, dev, snap, a, algo):
    """the same step on a fresh context without GP_CFG_ASYNC_SNAPSHOT"""
    f = gangpack.GangPacker()
    try:
        s = Step(torch, dev, max(int(a["off"][-1]), 1))
        s.put(s.upload(snap, a), torch.cuda.current_stream())
        torch.cuda.synchronize()
        s.snapshot(f)
        s.pack(f, algo)
        return s.result(f, a)
    finally:
        f.close()


def assert_same(got, want, what):
    assert np.array_equal(got[0], want[0]), (what, "DriverNode")
    assert np.array_equal(got[1], want[1]), (what, "ExecutorNodes")
    assert got[2] == want[2], (what, "statistics", got[2], want[2])


def cases(seed):
    rng = np.random.default_rng(seed)
    out = []
    for r in range(2):                      # twice round, in another order: each step follows a different layout
        for i in rng.permutation(len(SIZES) * 3):
            sizes, kind = SIZES[i % len(SIZES)], i // len(SIZES)
            out.append((snapshot(rng, sizes, kind), apps(rng)))
    return out


@pytest.mark.parametrize("algo", [0, 1])
def test_graph_replays_across_changing_snapshots(gangpack, algo):
    """The step captured once into a CUDA graph; before every replay the snapshot and application tensors are rewritten
    on the library's stream."""
    import torch
    dev = torch.device("cuda", 0)
    steps = cases(11 + algo)
    want = [reference(gangpack, torch, dev, snap, a, algo) for snap, a in steps]
    p = gangpack.GangPacker(async_snapshot=True)
    try:
        stream = torch.cuda.ExternalStream(p.stream_handle(), device=dev)
        s = Step(torch, dev, max(int(a["off"][-1]) for _, a in steps))
        on_dev = [s.upload(snap, a) for snap, a in steps]
        torch.cuda.synchronize()
        s.put(on_dev[0], stream)
        with torch.cuda.stream(stream):
            for _ in range(2):
                s.snapshot(p)
                s.pack(p, algo)
            p.stats()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                s.snapshot(p)
                s.pack(p, algo)
            for j, (_, a) in enumerate(steps):
                s.put(on_dev[j], stream)
                s.d.fill_(-7); s.e.fill_(-7)
                graph.replay()
                assert_same(s.result(p, a), want[j], f"replay {j}")
    finally:
        p.close()


@pytest.mark.parametrize("algo", [0, 1])
def test_eager_steps_and_pack_after_pack(gangpack, algo):
    """The same steps issued one call at a time.  Each snapshot call is followed by two pack calls on the same inputs
    (the second follows a pack call, not the layout, and waits for everything before it)."""
    import torch
    dev = torch.device("cuda", 0)
    steps = cases(21 + algo)
    want = [reference(gangpack, torch, dev, snap, a, algo) for snap, a in steps]
    cap = max(int(a["off"][-1]) for _, a in steps)
    p = gangpack.GangPacker(async_snapshot=True)
    try:
        stream = torch.cuda.ExternalStream(p.stream_handle(), device=dev)
        s, s2 = Step(torch, dev, cap), Step(torch, dev, cap)
        on_dev = [s.upload(snap, a) for snap, a in steps]
        torch.cuda.synchronize()
        for j, (_, a) in enumerate(steps):
            s.put(on_dev[j], stream)
            with torch.cuda.stream(stream):
                s.d.fill_(-7); s.e.fill_(-7); s2.d.fill_(-7); s2.e.fill_(-7)
            s2.ta = s.ta
            s.snapshot(p)
            s.pack(p, algo)
            s2.pack(p, algo)
            second = s2.result(p, a)
            assert_same(second, want[j], f"step {j}, second pack")
            first = s.result(p, a)
            assert np.array_equal(first[0], want[j][0]) and np.array_equal(first[1], want[j][1]), f"step {j}, first pack"
    finally:
        p.close()
