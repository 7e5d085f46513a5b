"""The C++ host layer's extender::ResidentDrivers and FitEarlierDriversDriverTable (tests/host_resident_drivers_test.cpp):
pending-driver pod events with capacities that double and replay, then the driver-table FIFO step against the per-call
recipe (FilterToEarliestAndSort + FitEarlierDrivers) on the same pods -- including a driver table reset behind the host's
back, refused, replayed and answered by the per-call path."""
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
    return os.path.join(HOST, "host_resident_drivers_test")


def test_host_resident_drivers_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_resident_drivers(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_resident_drivers_test: all passed" in p.stdout
