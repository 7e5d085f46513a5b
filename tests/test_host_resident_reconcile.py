"""The C++ host layer's resident reconciler and marker (tests/host_resident_reconcile_test.cpp): extender::ReconcileFindNodesResident
and UnschedulablePodMarker's resident sweep, each flushing its tables once and making one device call, against the per-call host
entries on a restatement of the same ResourceReservation, soft-store and pod events -- a refused update and its replay included."""
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
    return os.path.join(HOST, "host_resident_reconcile_test")


def test_host_resident_reconcile_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_resident_reconcile(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_resident_reconcile_test: all passed" in p.stdout
