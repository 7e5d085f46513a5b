"""CPU-only checks of gp_pack_fifo_zones_groups' boundary: the gp_instance_groups ctypes mirror against a C compiler's view
of include/gangpack.h, how GangPacker.pack_fifo_zones_groups marshals its arguments (through a fake library), and a
pure-Python model of how the call splits the queue into per-instance-group queues and scratch rows."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import k8s_spark_scheduler_b200 as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
native = g.native


def test_instance_groups_layout_matches_header():
    fields = [f for f, _ in native.gp_instance_groups._fields_]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "gangpack.h"\nint main(void) {\n  printf("%zu'
    src += " %zu" * len(fields) + '\\n", sizeof(gp_instance_groups)'
    src += "".join(", offsetof(gp_instance_groups, %s)" % f for f in fields) + ");\n  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    s = native.gp_instance_groups
    assert got == [C.sizeof(s)] + [getattr(s, f).offset for f in fields]


def _arr(addr, ctype, n):
    return None if not addr else np.ctypeslib.as_array((ctype * n).from_address(addr)).copy()


class FakeLib:
    """Stands in for libgangpack.so: records what gp_pack_fifo_zones_groups receives while the call runs."""

    def __init__(self):
        self.seen = None

    def __getattr__(self, name):
        if not name.startswith("gp_"):
            raise AttributeError(name)

        def call(*args):
            if name == "gp_pack_fifo_zones_groups":
                _, a, packer, mode, ig, r = args
                a, ig, r = a._obj, ig._obj, r._obj
                G = ig.n_instance_groups
                q = a.n_apps
                e_n = int(_arr(ig.exec_off, C.c_int32, G + 1)[-1]) if ig.exec_off else 0
                d_n = int(_arr(ig.drv_off, C.c_int32, G + 1)[-1]) if ig.drv_off else 0
                self.seen = dict(packer=packer, mode=mode, G=G, group_off=_arr(ig.group_off, C.c_int32, G + 1),
                                 n_zones=_arr(ig.n_zones, C.c_int32, G), exec_off=_arr(ig.exec_off, C.c_int32, G + 1),
                                 exec_order=_arr(ig.exec_order, C.c_int32, e_n), drv_off=_arr(ig.drv_off, C.c_int32, G + 1),
                                 drv_order=_arr(ig.drv_order, C.c_int32, d_n), group=_arr(a.group, C.c_int32, q),
                                 skip=_arr(a.skip_if_no_fit, C.c_uint8, q), count=_arr(a.exe_count, C.c_int32, q),
                                 cap=r.executor_nodes_cap, out_null=[not r.zone, not r.driver_node, not r.avg_efficiency])
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(native, "_lib", f)
    return f


def _apps(q, group=None, young=None):
    a = {k: np.arange(q, dtype=np.int64) for k in ("drv_cpu", "drv_mem", "exe_cpu", "exe_mem")}
    a["count"] = np.arange(q, dtype=np.int32) % 3
    if group is not None:
        a["group"] = group
    if young is not None:
        a["young"] = young
    return a


def test_marshal_single_az(fake):
    p = native.GangPacker()
    apps = _apps(5, group=[1, 0, 1, 2, 0], young=[1, 0, 0, 1, 0])
    zone, drv, exe, off, avg = p.pack_fifo_zones_groups(apps, native.BP_SINGLE_AZ_TIGHTLY_PACK, 2, [0, 2, 5, 6])
    s = fake.seen
    assert (s["packer"], s["mode"], s["G"]) == (native.BP_SINGLE_AZ_TIGHTLY_PACK, 2, 3)
    assert list(s["group_off"]) == [0, 2, 5, 6] and list(s["group"]) == [1, 0, 1, 2, 0] and list(s["skip"]) == [1, 0, 0, 1, 0]
    assert s["n_zones"] is None and s["exec_off"] is None and s["exec_order"] is None and s["drv_off"] is None and s["drv_order"] is None
    assert s["cap"] == max(int(off[-1]), 1) and s["out_null"] == [False, False, False]
    assert len(zone) == len(drv) == 5 and avg.shape == (5, 4)


def test_marshal_az_aware_and_default_group(fake):
    p = native.GangPacker()
    p.pack_fifo_zones_groups(_apps(3), native.BP_AZ_AWARE_TIGHTLY_PACK, 1, np.array([0, 2, 3], np.int64), n_zones=[1, 0],
                             exec_off=[0, 3, 4], exec_order=[5, 1, 2, 0], drv_off=[0, 1, 3], drv_order=[2, 3, 0])
    s = fake.seen
    assert s["G"] == 2 and list(s["n_zones"]) == [1, 0]
    assert list(s["exec_off"]) == [0, 3, 4] and list(s["exec_order"]) == [5, 1, 2, 0]
    assert list(s["drv_off"]) == [0, 1, 3] and list(s["drv_order"]) == [2, 3, 0]
    assert s["group"] is None and s["skip"] is None                       # NULL group: every application in instance group 0


def queue_split(group, count, n_zones, az):
    """Model of the call's host pass: a stable counting sort of the application indices by instance group, and per instance
    group its queue range, row pitch (largest exe_count, at least 1, rounded up to 4) and scratch rows
    ((n_zones + az) x pitch).  -> (queue, [(q_begin, q_end, row_base, row_pitch)], total rows)."""
    G = len(n_zones)
    n = [0] * G
    pitch = [0] * G
    for b, k in zip(group, count):
        n[b] += 1
        pitch[b] = max(pitch[b], max(int(k), 0))
    desc, qb, rows = [], 0, 0
    for b in range(G):
        p = (max(pitch[b], 1) + 3) & ~3
        desc.append([qb, qb, rows, p])
        qb += n[b]
        rows += (n_zones[b] + az) * p
    queue = [0] * len(group)
    for i, b in enumerate(group):
        queue[desc[b][1]] = i
        desc[b][1] += 1
    return queue, [tuple(d) for d in desc], rows


@pytest.mark.parametrize("seed", range(6))
def test_queue_split_model(seed):
    rng = np.random.default_rng(seed)
    G = int(rng.integers(1, 20))
    q = int(rng.integers(0, 300))
    group = rng.integers(0, G, q)
    count = np.where(rng.random(q) < 0.1, rng.integers(20, 200, q), rng.integers(-2, 12, q))
    n_zones = rng.integers(0, 65, G)
    for az in (0, 1):
        queue, desc, rows = queue_split(group, count, n_zones, az)
        for b, (lo, hi, base, p) in enumerate(desc):
            assert queue[lo:hi] == [i for i in range(q) if group[i] == b]          # its applications, in queue order
            mine = count[group == b]
            assert p % 4 == 0 and p >= max([1] + list(mine)) and p < max([1] + list(mine)) + 4
            nxt = desc[b + 1][2] if b + 1 < G else rows
            assert nxt - base == (n_zones[b] + az) * p                            # rows never overlap
        assert sorted(queue) == list(range(q))
        # the scratch is bounded by the batch's own ExecutorNodes (each pitch <= its group's largest count + 4), not by
        # G x the batch-wide maximum
        assert rows <= (64 + az) * (int(np.maximum(count, 0).sum()) + 4 * G)
