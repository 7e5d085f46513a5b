"""metrics::PlacementMetrics in the C++ host layer against a string-keyed C++ literal of the three placement reporters
(tests/host_placement_metrics_test.cpp): one gp_placement_metrics call per placement, equal on every field."""
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
    return os.path.join(HOST, "host_placement_metrics_test")


def test_host_placement_metrics_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_placement_metrics_against_literal(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "all passed" in p.stdout
