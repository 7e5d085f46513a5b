"""The ctypes mirrors of the resident reservation table's structs (gp_reservation_table_size, gp_reservation_delta,
gp_resident_usage) against a C compiler's view of include/gangpack.h: sizes and every field's offset."""
import ctypes
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reservation_table_struct_layout_matches_header():
    from k8s_spark_scheduler_b200 import native
    structs = {"gp_reservation_table_size": native.gp_reservation_table_size, "gp_reservation_delta": native.gp_reservation_delta,
               "gp_resident_usage": native.gp_resident_usage}
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
