"""binpack::AzAwareTightlyPack in the C++ host layer against the oracle's az-aware packer (tests/host_az_aware_batch_test.cpp):
one gp_pack_batch_az_aware call per decision, the undivided fallback included, up to 70 candidate zones."""
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
    return os.path.join(HOST, "host_az_aware_batch_test")


def test_host_az_aware_batch_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_az_aware_batch_against_oracle(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "all passed" in p.stdout
