"""CPU-only checks of gp_prepare_cluster_groups and gp_packing_efficiency_groups at the boundary: the
gp_instance_group_orders ctypes mirror against a C compiler's view of include/gangpack.h, how GangPacker.prepare_cluster_groups
and packing_efficiency_groups marshal their arguments (through a fake library), and that both symbols are exported, bound
and documented."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import k8s_spark_scheduler_b200 as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
native = g.native


def test_instance_group_orders_matches_header():
    fields = [f for f, _ in native.gp_instance_group_orders._fields_]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "gangpack.h"\nint main(void) {\n  printf("%zu'
    src += " %zu" * len(fields) + '\\n", sizeof(gp_instance_group_orders)'
    src += "".join(", offsetof(gp_instance_group_orders, %s)" % f for f in fields) + ");\n  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    s = native.gp_instance_group_orders
    assert got == [C.sizeof(s)] + [getattr(s, f).offset for f in fields]


def _arr(addr, ctype, n):
    return None if not addr else np.ctypeslib.as_array((ctype * n).from_address(addr)).copy()


class FakeLib:
    """Stands in for libgangpack.so: records the arguments and writes a small two-instance-group result back."""

    def __init__(self):
        self.seen = {}

    def __getattr__(self, name):
        if not name.startswith("gp_"):
            raise AttributeError(name)

        def call(*args):
            if name == "gp_prepare_cluster_groups":
                _, ui, si, ig, G, o = args
                ui, si, o = ui._obj, si._obj, o._obj
                n = ui.n_nodes
                self.seen[name] = dict(n=n, G=G, ig=_arr(ig, C.c_int32, n), zone_id=_arr(si.zone_id, C.c_int32, n),
                                       n_zones=si.n_zones, ptrs={f: bool(getattr(o, f)) for f, _ in o._fields_[2:]})
                o.n_driver, o.n_executor = 2, 3
                for f, v in (("exec_off", [0, 2, 3]), ("drv_off", [0, 1, 2]), ("exec_order", [3, 0, 1]), ("drv_order", [0, 2]),
                             ("undefined_ties", [1, 0])):
                    p = getattr(o, f)
                    if p:
                        C.memmove(p, np.array(v, np.int32).ctypes.data, 4 * len(v))
                C.c_int32.from_address(si.undefined_ties).value = 1
            elif name == "gp_packing_efficiency_groups":
                _, a, algo, r, charged, ig, G, avg = args
                a, r = a._obj, r._obj
                q = a.n_apps
                self.seen[name] = dict(algo=algo, charged=charged, G=G, ig=_arr(ig, C.c_int32, 4), group=_arr(a.group, C.c_int32, q),
                                       driver=_arr(r.driver_node, C.c_int32, q), cap=r.executor_nodes_cap)
                C.memmove(avg, np.arange(4 * q, dtype=np.float64).ctypes.data, 32 * q)
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(native, "_lib", f)
    return f


def _usage(n):
    z = np.zeros(n, np.int64)
    return [z + 4000, z + (1 << 32), z], None, np.zeros(0, np.int32), [np.zeros(0, np.int64)] * 3


def test_marshal_prepare_groups(fake):
    p = native.GangPacker()
    out = p.prepare_cluster_groups(*_usage(4), [0, 1, 0, -1], 2, zone_id=[0, 1, 1, 0], n_zones=2)
    s = fake.seen["gp_prepare_cluster_groups"]
    assert (s["n"], s["G"], s["n_zones"]) == (4, 2, 2)
    assert list(s["ig"]) == [0, 1, 0, -1] and list(s["zone_id"]) == [0, 1, 1, 0]
    assert all(s["ptrs"].values())
    assert (out["n_driver"], out["n_executor"], out["undefined_ties"]) == (2, 3, 1)
    assert list(out["exec_off"]) == [0, 2, 3] and list(out["drv_off"]) == [0, 1, 2] and list(out["ig_undefined_ties"]) == [1, 0]
    assert list(out["exec_order"]) == [3, 0, 1] and list(out["drv_order"]) == [0, 2]


def test_marshal_prepare_groups_without_orders(fake):
    p = native.GangPacker()
    out = p.prepare_cluster_groups(*_usage(3), None, 1, orders=False)
    s = fake.seen["gp_prepare_cluster_groups"]
    assert s["ig"] is None and s["G"] == 1
    assert [k for k, v in s["ptrs"].items() if v] == ["undefined_ties"]
    assert "exec_order" not in out and "exec_off" not in out


def test_marshal_efficiency_groups(fake):
    p = native.GangPacker()
    apps = {k: np.arange(3, dtype=np.int64) for k in ("drv_cpu", "drv_mem", "exe_cpu", "exe_mem")}
    apps["count"] = np.array([1, 0, 2], np.int32); apps["group"] = [1, 0, 1]
    placed = (np.array([2, -1, 3], np.int32), np.array([2, 3, 3], np.int32), np.array([0, 1, 1, 3], np.int64))
    avg = p.packing_efficiency_groups(apps, placed, native.DISTRIBUTE_EVENLY, [0, 0, 1, 1], 2, charged=native.MODE_FIFO_EXACT)
    s = fake.seen["gp_packing_efficiency_groups"]
    assert (s["algo"], s["charged"], s["G"], s["cap"]) == (native.DISTRIBUTE_EVENLY, native.MODE_FIFO_EXACT, 2, 3)
    assert list(s["ig"]) == [0, 0, 1, 1] and list(s["group"]) == [1, 0, 1] and list(s["driver"]) == [2, -1, 3]
    assert avg.shape == (3, 4) and avg[2, 3] == 11.0


def test_entries_exported_bound_and_documented():
    g.native.build()
    out = subprocess.check_output(["nm", "-D", "--defined-only", g.native.LIB_PATH], text=True)
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = g.native.load()
    assert L.gp_prepare_cluster_groups.argtypes[-1]._type_ is g.native.gp_instance_group_orders
    assert len(L.gp_packing_efficiency_groups.argtypes) == 8
    for sym in ("gp_prepare_cluster_groups", "gp_packing_efficiency_groups"):
        assert sym in g.native.EXPORTS and sym in defined, sym
        for doc in ("include/gangpack.h", "DESIGN.md", "INTEGRATION.md", "README.md"):
            assert sym in open(os.path.join(ROOT, doc)).read(), (sym, doc)
