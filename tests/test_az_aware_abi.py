"""CPU-only checks of gp_pack_fifo_az_aware's boundary: the gp_az_orders ctypes mirror against a C compiler's view of
include/gangpack.h, and the az-aware instantiations of the zone FIFO kernel inside libgangpack.so."""
import ctypes
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    import k8s_spark_scheduler_b200 as g
    g.native.build()
    return g.native


def test_az_orders_layout_matches_header(native):
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gangpack.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu %zu\n", sizeof(gp_az_orders), offsetof(gp_az_orders, n_zones), offsetof(gp_az_orders, n_exec),
             offsetof(gp_az_orders, exec_order), offsetof(gp_az_orders, n_drv), offsetof(gp_az_orders, drv_order));
      return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    o = native.gp_az_orders
    assert got == [ctypes.sizeof(o), o.n_zones.offset, o.n_exec.offset, o.exec_order.offset, o.n_drv.offset, o.drv_order.offset]


def test_library_contains_the_az_aware_kernels(native):
    """gp_pack_fifo_zones_cta<3, FIFO_MODE, GatherSlots> for both accounting modes, and the kernel that builds the
    fallback view"""
    out = subprocess.check_output(["cuobjdump", "-sass", native.LIB_PATH], text=True)
    names = subprocess.run(["c++filt"], input="\n".join(l.split(":", 1)[1].strip() for l in out.splitlines() if "Function :" in l),
                           capture_output=True, text=True, check=True).stdout.splitlines()
    for mode in (1, 2):
        assert any(n.startswith("void gp::gp_pack_fifo_zones_cta<3, %d, gp::GatherSlots>(" % mode) for n in names), mode
    assert any(n.startswith("gp::gp_build_fallback_view(") for n in names)
