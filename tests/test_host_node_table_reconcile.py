"""The C++ host layer's extender::ReconcileFindNodesNodeTable and UnschedulablePodMarker's node-table sweeps
(tests/host_node_table_reconcile_test.cpp): node events with creation times over the four resident tables, then each
node-table path against the resident host path on the host's own columns -- including an unlisted instance group and a node
table reset behind the host's back, both refused, replayed and answered."""
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
    return os.path.join(HOST, "host_node_table_reconcile_test")


def test_host_node_table_reconcile_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_node_table_reconcile(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_node_table_reconcile_test: all passed" in p.stdout
