"""extender::FitEarlierDrivers("az-aware-tightly-pack") in the C++ host layer against the oracle's FIFO loop
(tests/host_az_aware_test.cpp): one gp_pack_fifo_az_aware call per queue, the per-driver loop above 64 zones."""
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
    return os.path.join(HOST, "host_az_aware_test")


def test_host_az_aware_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_az_aware_fifo_against_oracle(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "all passed" in p.stdout
