"""The C++ host layer's UnschedulablePodMarker driver-table scan (tests/host_resident_marker_test.cpp): node and
pending-driver pod events, then the scan from the driver table against the per-call node-table affinity sweep over the
same stale drivers -- including a stale driver's affinity id rewritten out of range behind the host's back, refused,
replayed and answered by the per-call path."""
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
    return os.path.join(HOST, "host_resident_marker_test")


def test_host_resident_marker_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_resident_marker(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_resident_marker_test: all passed" in p.stdout
