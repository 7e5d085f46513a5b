"""extender::ReconcileFindNodes in the C++ host layer against the string-keyed C literal of the failover reconciler
(tests/host_reconcile_test.cpp over tests/reconcile_oracle.c), with nodes and drivers that carry no instance-group label."""
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
    return os.path.join(HOST, "host_reconcile_test")


def test_host_reconcile_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_reconcile_against_the_literal(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "all passed" in p.stdout
