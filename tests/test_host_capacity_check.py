"""extender::UnschedulablePodMarker::DoesPodsExceedClusterCapacity in the C++ host layer against the per-driver
DoesPodExceedClusterCapacity path of the same layer (tests/host_capacity_check_test.cpp): one gp_exceeds_cluster_capacity
call per sweep against each packer's BinpackFunc on the driver's zero-usage metadata, for all five packers."""
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
    return os.path.join(HOST, "host_capacity_check_test")


def test_host_capacity_check_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_capacity_check_against_per_driver_binpack(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "all passed" in p.stdout
