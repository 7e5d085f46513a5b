"""The C++ host layer's affinity interning, affinity::MatchRequiredNodeAffinity and the UnschedulablePodMarker overload over
affinity programs (tests/host_affinity_marker_test.cpp): reference quirks by hand, and the overlapping-set sweep against the
one-class-per-node overload called per affinity, for all five packers."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-spark-scheduler_b200", "host")


@pytest.fixture(scope="module")
def host_binary():
    import k8s_spark_scheduler_b200 as g
    g.native.build()
    subprocess.check_call(["make", "-C", HOST, "-s"])
    return os.path.join(HOST, "host_affinity_marker_test")


def test_host_affinity_marker_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_affinity_marker(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_affinity_marker_test: all passed" in p.stdout
