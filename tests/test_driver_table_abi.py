"""The ctypes mirrors of the resident driver table's structs (gp_driver_table_size, gp_driver_delta, gp_driver_queue) against
a C compiler's view of include/gangpack.h, and the new entries declared, exported, bound and documented."""
import ctypes
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["gp_driver_table_reset", "gp_driver_table_update", "gp_pack_fifo_driver_table", "gp_pack_fifo_zones_groups_driver_table"]


def test_driver_table_struct_layout_matches_header():
    from k8s_spark_scheduler_b200 import native
    structs = {"gp_driver_table_size": native.gp_driver_table_size, "gp_driver_delta": native.gp_driver_delta,
               "gp_driver_queue": native.gp_driver_queue}
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


def test_driver_table_entries_exported_bound_and_documented():
    import k8s_spark_scheduler_b200 as g
    g.native.build()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gangpack.h")).read(), flags=re.S)
    out = subprocess.check_output(["nm", "-D", "--defined-only", g.native.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    lib = g.native.load()
    docs = {f: open(os.path.join(ROOT, f)).read() for f in ("INTEGRATION.md", "DESIGN.md", "README.md")}
    for s in ENTRIES:
        assert re.search(rf"\b{s}\s*\(", header), s
        assert s in g.native.EXPORTS and s in exported, s
        assert getattr(lib, s).restype is ctypes.c_int and getattr(lib, s).argtypes, s
        for name, text in docs.items():
            assert s in text, (s, name)
