"""gp_node_delta with its creation column against a C compiler's view of include/gangpack.h, and the node-table forms of the
failover reconciler and the unschedulable-pod marker declared, exported, bound and documented."""
import ctypes
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["gp_reconcile_find_nodes_node_table", "gp_exceeds_cluster_capacity_node_table",
           "gp_exceeds_cluster_capacity_affinity_node_table"]


def test_node_delta_layout_with_creation_matches_header():
    from k8s_spark_scheduler_b200 import native
    cls = native.gp_node_delta
    assert cls._fields_[-1][0] == "creation"
    lines = ['printf("%zu\\n", sizeof(gp_node_delta));'] + [f'printf("%zu\\n", offsetof(gp_node_delta, {f}));' for f, _ in cls._fields_]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"gangpack.h\"\nint main(void) {\n" + "\n".join(lines) + "\nreturn 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "t.c"), os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert got == [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]


def test_entries_exported_bound_and_documented():
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
    for m in ("reconcile_find_nodes_node_table", "exceeds_cluster_capacity_node_table", "exceeds_cluster_capacity_affinity_node_table"):
        assert callable(getattr(g.native.GangPacker, m)), m
