"""The resident reconciler and marker entries (gp_reconcile_find_nodes_resident, gp_exceeds_cluster_capacity_resident,
gp_exceeds_cluster_capacity_affinity_resident): exported by the library, and the ctypes argument lists the binding gives them
checked against a C compiler's view of include/gangpack.h -- each parameter's type, and the layout of the structs it points to."""
import ctypes
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the C type of each ctypes argument the binding declares; a struct pointer names its struct
C_OF = {ctypes.c_void_p: "void*", ctypes.c_int: "int", ctypes.c_int32: "int32_t"}
ENTRIES = {
    "gp_reconcile_find_nodes_resident": ["gp_ctx*", "const gp_resident_usage*", "const gp_reconcile_nodes*", "const gp_apps*",
                                         "gp_reconcile_results*"],
    "gp_exceeds_cluster_capacity_resident": ["gp_ctx*", "const gp_capacity_nodes*", "const int32_t*", "const gp_apps*", "gp_binpacker",
                                             "uint8_t*"],
    "gp_exceeds_cluster_capacity_affinity_resident": ["gp_ctx*", "const gp_capacity_nodes*", "const int32_t*", "const gp_node_labels*",
                                                      "const gp_node_affinities*", "const gp_apps*", "gp_binpacker", "uint8_t*", "uint8_t*"],
}


def test_exported_and_listed():
    from k8s_spark_scheduler_b200 import native
    for name in ENTRIES:
        assert name in native.EXPORTS
    header = open(os.path.join(ROOT, "include", "gangpack.h")).read()
    for name in ENTRIES:
        assert f"gp_status {name}(" in header


def test_argument_lists_match_header():
    """the header's prototypes have exactly the parameter types above (checked at compile time), and the binding passes one ctypes argument of the matching kind and size for each"""
    from k8s_spark_scheduler_b200 import native
    L = native.load()
    checks = []
    for name, params in ENTRIES.items():
        checks.append(f"_Static_assert(__builtin_types_compatible_p(__typeof__(&{name}), gp_status (*)({', '.join(params)})), "
                      f"\"{name}\");")
        argtypes = getattr(L, name).argtypes
        assert len(argtypes) == len(params), name
        for t, c in zip(argtypes, params):
            if c.endswith("*"):
                assert t is ctypes.c_void_p or issubclass(t, ctypes._Pointer), (name, c, t)
                if issubclass(t, ctypes._Pointer):
                    assert c.rstrip("*").split()[-1] == t._type_.__name__, (name, c, t)
            else:
                assert t is ctypes.c_int and c in ("gp_binpacker", "int"), (name, c, t)
    structs = {"gp_resident_usage": native.gp_resident_usage, "gp_reconcile_nodes": native.gp_reconcile_nodes,
               "gp_reconcile_results": native.gp_reconcile_results, "gp_capacity_nodes": native.gp_capacity_nodes}
    lines = [f'printf("%zu\\n", sizeof(gp_binpacker));']
    for sname, cls in structs.items():
        lines.append(f'printf("%zu\\n", sizeof({sname}));')
        lines += [f'printf("%zu\\n", offsetof({sname}, {f}));' for f, _ in cls._fields_]
    src = ("#include <stdio.h>\n#include <stddef.h>\n#include \"gangpack.h\"\nint main(void) {\n" + "\n".join(checks + lines) +
           "\nreturn 0; }\n")
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "t.c"), os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    want = [ctypes.sizeof(ctypes.c_int)]
    for cls in structs.values():
        want.append(ctypes.sizeof(cls))
        want += [getattr(cls, f).offset for f, _ in cls._fields_]
    assert got == want
