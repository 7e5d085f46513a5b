"""CPU-only checks of gp_placement_metrics[_device] at the boundary: the gp_placement_record ctypes mirror (and the numpy
dtype the binding returns) against a C compiler's view of include/gangpack.h, how GangPacker.placement_metrics marshals its
arguments (through a fake library), and that both symbols are exported, bound and documented."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import k8s_spark_scheduler_b200 as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
native = g.native


def test_placement_record_matches_header():
    fields = [f for f, _ in native.gp_placement_record._fields_]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "gangpack.h"\nint main(void) {\n  printf("%zu'
    src += " %zu" * len(fields) + '\\n", sizeof(gp_placement_record)'
    src += "".join(", offsetof(gp_placement_record, %s)" % f for f in fields) + ");\n  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    s = native.gp_placement_record
    assert got == [C.sizeof(s)] + [getattr(s, f).offset for f in fields] == [32, 0, 4, 8, 12, 16, 24]
    d = native.PLACEMENT_DTYPE
    assert d.itemsize == got[0] and [d.fields[f][1] for f in fields] == got[1:]


def _arr(addr, ctype, n):
    return None if not addr else np.ctypeslib.as_array((ctype * n).from_address(addr)).copy()


class FakeLib:
    """Stands in for libgangpack.so: records the arguments and writes one record per row back."""

    def __init__(self):
        self.seen = {}

    def __getattr__(self, name):
        if not name.startswith("gp_"):
            raise AttributeError(name)

        def call(*args):
            if name == "gp_placement_metrics":
                _, a, r, n, zone, nz, ig, G, out = args
                a, r = a._obj, r._obj
                q = a.n_apps
                self.seen[name] = dict(n=n, nz=nz, G=G, zone=_arr(zone, C.c_int32, n), ig=_arr(ig, C.c_int32, n),
                                       count=_arr(a.exe_count, C.c_int32, q), group=_arr(a.group, C.c_int32, q),
                                       off=_arr(a.exec_out_off, C.c_int64, q + 1), driver=_arr(r.driver_node, C.c_int32, q),
                                       cap=r.executor_nodes_cap)
                rec = (native.gp_placement_record * q).from_address(out)
                for i in range(q):
                    rec[i] = native.gp_placement_record(i - 1, 2 * i, 3 * i, 4 * i, 1 << 40, -i)
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(native, "_lib", f)
    return f


def test_marshal_placement_metrics(fake):
    p = native.GangPacker()
    apps = {"count": np.array([1, 0, 2], np.int32), "group": [1, 0, 1], "off": [0, 1, 1, 3]}
    placed = (np.array([2, -1, 3], np.int32), np.array([2, 3, 3], np.int32), np.array([0, 1, 1, 3], np.int64))
    rec = p.placement_metrics(apps, placed, [0, 2, 1, 2], instance_group=[0, 0, 1, 1], n_instance_groups=2)
    s = fake.seen["gp_placement_metrics"]
    assert (s["n"], s["nz"], s["G"], s["cap"]) == (4, 3, 2, 3)
    assert list(s["zone"]) == [0, 2, 1, 2] and list(s["ig"]) == [0, 0, 1, 1] and list(s["group"]) == [1, 0, 1]
    assert list(s["count"]) == [1, 0, 2] and list(s["off"]) == [0, 1, 1, 3] and list(s["driver"]) == [2, -1, 3]
    assert rec.dtype == native.PLACEMENT_DTYPE and len(rec) == 3
    assert tuple(rec[2]) == (1, 4, 6, 8, 1 << 40, -2)


def test_marshal_one_group_and_explicit_zone_count(fake):
    p = native.GangPacker()
    rec = p.placement_metrics({"count": np.array([2], np.int32)}, ([1], [], [0, 2]), [0, 0, 0], n_metric_zones=3)
    s = fake.seen["gp_placement_metrics"]
    assert s["ig"] is None and s["group"] is None and s["nz"] == 3 and s["cap"] == 1 and len(rec) == 1


def test_entries_exported_bound_and_documented():
    g.native.build()
    out = subprocess.check_output(["nm", "-D", "--defined-only", g.native.LIB_PATH], text=True)
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = g.native.load()
    assert len(L.gp_placement_metrics.argtypes) == 9 and len(L.gp_placement_metrics_device.argtypes) == 11
    for sym in ("gp_placement_metrics", "gp_placement_metrics_device"):
        assert sym in g.native.EXPORTS and sym in defined, sym
        for doc in ("include/gangpack.h", "DESIGN.md", "INTEGRATION.md", "README.md"):
            assert sym in open(os.path.join(ROOT, doc)).read(), (sym, doc)
