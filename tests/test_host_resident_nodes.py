"""The C++ host layer's resources::ResidentNodes and NodeTableLabels (tests/host_resident_nodes_test.cpp): node add / update /
delete events with capacities that double and replay, node ids that are reused and name keys that run out of gaps, then the
node-table prepare and reschedule entries against the *_resident entries on the host's per-call columns of the same nodes --
including a node table reset behind the host's back, refused, replayed and answered again."""
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
    return os.path.join(HOST, "host_resident_nodes_test")


def test_host_resident_nodes_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_resident_nodes(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_resident_nodes_test: all passed" in p.stdout
