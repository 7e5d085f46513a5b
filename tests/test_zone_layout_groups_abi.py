"""CPU-only checks of gp_prepare_cluster_zones_groups' boundary: the gp_instance_group_layout ctypes mirror against a C
compiler's view of include/gangpack.h, how GangPacker.prepare_cluster_zones_groups and pack_fifo_zones_groups(groups=None)
marshal their arguments (through a fake library), and that the symbol is exported, bound and documented."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import k8s_spark_scheduler_b200 as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
native = g.native


def test_instance_group_layout_matches_header():
    fields = [f for f, _ in native.gp_instance_group_layout._fields_]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "gangpack.h"\nint main(void) {\n  printf("%zu'
    src += " %zu" * len(fields) + '\\n", sizeof(gp_instance_group_layout)'
    src += "".join(", offsetof(gp_instance_group_layout, %s)" % f for f in fields) + ");\n  return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    s = native.gp_instance_group_layout
    assert got == [C.sizeof(s)] + [getattr(s, f).offset for f in fields]


def _arr(addr, ctype, n):
    return None if not addr else np.ctypeslib.as_array((ctype * n).from_address(addr)).copy()


class FakeLib:
    """Stands in for libgangpack.so: records the arguments and writes a small two-instance-group layout back."""

    def __init__(self):
        self.seen = {}

    def __getattr__(self, name):
        if not name.startswith("gp_"):
            raise AttributeError(name)

        def call(*args):
            if name == "gp_prepare_cluster_zones_groups":
                _, ui, si, ig, G, lo = args
                ui, si, lo = ui._obj, si._obj, lo._obj
                n = ui.n_nodes
                self.seen[name] = dict(n=n, G=G, ig=_arr(ig, C.c_int32, n), kind=lo.kind, zone_id=_arr(si.zone_id, C.c_int32, n),
                                       n_zones=si.n_zones, ptrs={f: bool(getattr(lo, f)) for f, _ in lo._fields_[4:]})
                lo.n_groups, lo.n_driver, lo.n_executor = 3, 2, 3
                for f, v in (("group_off", [0, 2, 3]), ("n_zones", [1, 0]), ("exec_off", [0, 2, 3]), ("drv_off", [0, 1, 2]),
                             ("undefined_ties", [1, 0]), ("exec_order", [3, 0, 1]), ("drv_order", [0, 1]),
                             ("group_exec_off", [0, 1, 2, 3]), ("group_drv_off", [0, 1, 1, 2]), ("group_exec_order", [3, 0, 1]),
                             ("group_drv_order", [0, 1]), ("zone_of_group", [1, -1, -1])):
                    p = getattr(lo, f)
                    if p:
                        C.memmove(p, np.array(v, np.int32).ctypes.data, 4 * len(v))
                C.c_int32.from_address(si.undefined_ties).value = 1
            elif name == "gp_pack_fifo_zones_groups":
                _, a, packer, mode, ig, r = args
                self.seen[name] = dict(packer=packer, mode=mode, ig_null=ig is None, group=_arr(a._obj.group, C.c_int32, a._obj.n_apps))
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


def test_marshal_prepare(fake):
    p = native.GangPacker()
    out = p.prepare_cluster_zones_groups(*_usage(4), [0, 0, 1, -1], 2, zone_id=[0, 1, 1, 0], n_zones=2, kind=native.LAYOUT_SINGLE_AZ)
    s = fake.seen["gp_prepare_cluster_zones_groups"]
    assert (s["n"], s["G"], s["kind"], s["n_zones"]) == (4, 2, native.LAYOUT_SINGLE_AZ, 2)
    assert list(s["ig"]) == [0, 0, 1, -1] and list(s["zone_id"]) == [0, 1, 1, 0]
    assert all(s["ptrs"].values())
    assert (out["n_groups"], out["n_driver"], out["n_executor"], out["undefined_ties"]) == (3, 2, 3, 1)
    assert list(out["group_off"]) == [0, 2, 3] and list(out["n_zones"]) == [1, 0] and list(out["ig_undefined_ties"]) == [1, 0]
    assert list(out["exec_order"]) == [3, 0, 1] and list(out["drv_order"]) == [0, 1]
    assert list(out["group_exec_off"]) == [0, 1, 2, 3] and list(out["group_drv_order"]) == [0, 1]
    assert list(out["zone_of_group"]) == [1, -1, -1]


def test_marshal_prepare_without_layout_and_null_groups(fake):
    p = native.GangPacker()
    out = p.prepare_cluster_zones_groups(*_usage(3), None, 1, layout=False)
    s = fake.seen["gp_prepare_cluster_zones_groups"]
    assert s["ig"] is None and s["G"] == 1 and s["kind"] == native.LAYOUT_AZ_AWARE
    assert [k for k, v in s["ptrs"].items() if v] == ["group_off", "n_zones", "exec_off", "drv_off", "undefined_ties"]
    assert "exec_order" not in out and "zone_of_group" not in out


def test_marshal_fifo_groups_null(fake):
    p = native.GangPacker()
    apps = {k: np.arange(3, dtype=np.int64) for k in ("drv_cpu", "drv_mem", "exe_cpu", "exe_mem")}
    apps["count"] = np.array([1, 0, 2], np.int32); apps["group"] = [1, 0, 1]
    p.pack_fifo_zones_groups(apps, native.BP_AZ_AWARE_TIGHTLY_PACK, 2)
    s = fake.seen["gp_pack_fifo_zones_groups"]
    assert s["ig_null"] and (s["packer"], s["mode"]) == (native.BP_AZ_AWARE_TIGHTLY_PACK, 2) and list(s["group"]) == [1, 0, 1]
    p.pack_fifo_zones_groups(apps, native.BP_SINGLE_AZ_TIGHTLY_PACK, 1, group_off=[0, 1, 2])
    assert not fake.seen["gp_pack_fifo_zones_groups"]["ig_null"]


def test_entry_exported_bound_and_documented():
    g.native.build()
    assert "gp_prepare_cluster_zones_groups" in g.native.EXPORTS
    out = subprocess.check_output(["nm", "-D", "--defined-only", g.native.LIB_PATH], text=True)
    assert any(line.split()[-1] == "gp_prepare_cluster_zones_groups" for line in out.splitlines() if " T " in line)
    assert g.native.load().gp_prepare_cluster_zones_groups.argtypes[-1]._type_ is g.native.gp_instance_group_layout
    for doc in ("include/gangpack.h", "DESIGN.md", "INTEGRATION.md", "README.md"):
        assert "gp_prepare_cluster_zones_groups" in open(os.path.join(ROOT, doc)).read(), doc
