"""CPU-only checks of gp_pack_batch_az_aware's boundary: the exported symbol, the ctypes binding, the fallback kernels
inside libgangpack.so, and the host layer that calls it."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    import k8s_spark_scheduler_b200 as g
    g.native.build()
    return g.native


def test_symbol_exported_and_bound(native):
    out = subprocess.check_output(["nm", "-D", "--defined-only", native.LIB_PATH], text=True)
    assert re.search(r"\bT gp_pack_batch_az_aware$", out, re.M)
    assert "gp_pack_batch_az_aware" in native.EXPORTS
    f = native.load().gp_pack_batch_az_aware
    assert f.restype is ctypes.c_int
    assert f.argtypes == [ctypes.c_void_p, ctypes.POINTER(native.gp_apps), ctypes.POINTER(native.gp_az_orders),
                          ctypes.POINTER(native.gp_zone_results)]


def test_header_declares_it():
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gangpack.h")).read(), flags=re.S)
    assert re.search(r"gp_status gp_pack_batch_az_aware\(gp_ctx\* ctx, const gp_apps\* apps\s*, const gp_az_orders\* orders,\s*"
                     r"gp_zone_results\* out\);", header)


def test_library_contains_the_fallback_kernels(native):
    out = subprocess.check_output(["cuobjdump", "-sass", native.LIB_PATH], text=True)
    names = subprocess.run(["c++filt"], input="\n".join(l.split(":", 1)[1].strip() for l in out.splitlines() if "Function :" in l),
                           capture_output=True, text=True, check=True).stdout.splitlines()
    assert any(n.startswith("gp::gp_pack_az_fallback(") for n in names)
    assert any(n.startswith("gp::gp_az_fallback_list(") for n in names)
    assert "sm_90a" in subprocess.check_output(["cuobjdump", "-lelf", native.LIB_PATH], text=True)


def test_host_layer_calls_it_and_product_never_imports_the_oracle():
    host = open(os.path.join(ROOT, "k8s-spark-scheduler_b200", "host", "gangpack_host.hpp")).read()
    assert "gp_pack_batch_az_aware(" in host and "AzAwareLayout(" in host
    shim = open(os.path.join(ROOT, "k8s-spark-scheduler_b200", "go", "binpacker_gpu.go")).read()
    assert "C.gp_pack_batch_az_aware(" in shim
    pkg = os.path.join(ROOT, "k8s-spark-scheduler_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp", ".go")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert not re.search(r"(from|import)\s+oracle|gangpack_oracle|oracle/", text), f
