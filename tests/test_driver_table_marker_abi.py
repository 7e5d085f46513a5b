"""The ctypes mirrors of gp_stale_sweep and of gp_driver_delta (with its affinity column) against a C compiler's view of
include/gangpack.h, and gp_exceeds_cluster_capacity_driver_table declared, exported, bound and documented."""
import ctypes
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = "gp_exceeds_cluster_capacity_driver_table"


def test_stale_sweep_layout_matches_header():
    from k8s_spark_scheduler_b200 import native
    structs = {"gp_stale_sweep": native.gp_stale_sweep, "gp_driver_delta": native.gp_driver_delta}
    lines = []
    for name, cls in structs.items():
        lines.append(f'printf("%zu\\n", sizeof({name}));')
        lines += [f'printf("%zu\\n", offsetof({name}, {f}));' for f, _ in cls._fields_]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"gangpack.h\"\nint main(void) {\n" + "\n".join(lines) + "\nreturn 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "t.c"), os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    want = []
    for cls in structs.values():
        want.append(ctypes.sizeof(cls))
        want += [getattr(cls, f).offset for f, _ in cls._fields_]
    assert got == want
    assert native.gp_driver_delta._fields_[-1][0] == "affinity"        # appended: the earlier fields keep their offsets


def test_sweep_entry_exported_bound_and_documented():
    import k8s_spark_scheduler_b200 as g
    g.native.build()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gangpack.h")).read(), flags=re.S)
    out = subprocess.check_output(["nm", "-D", "--defined-only", g.native.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    lib = g.native.load()
    assert re.search(rf"\b{ENTRY}\s*\(", header)
    assert ENTRY in g.native.EXPORTS and ENTRY in exported
    assert getattr(lib, ENTRY).restype is ctypes.c_int and getattr(lib, ENTRY).argtypes
    for f in ("INTEGRATION.md", "DESIGN.md", "README.md"):
        assert ENTRY in open(os.path.join(ROOT, f)).read(), f
    assert hasattr(g.GangPacker, "exceeds_cluster_capacity_driver_table")
