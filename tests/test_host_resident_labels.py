"""The C++ host layer's affinity::ResidentLabels (tests/host_resident_labels_test.cpp): node add / relabel / delete events,
with capacities that double and replay and node ids that are reused, then the resident MatchRequiredNodeAffinity and
UnschedulablePodMarker's affinity sweep over both resident tables, against the per-call host paths on the same nodes --
including a refused resident call that replays the table and falls back to the per-call path."""
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
    return os.path.join(HOST, "host_resident_labels_test")


def test_host_resident_labels_binary_builds(host_binary):
    assert os.access(host_binary, os.X_OK)


@pytest.mark.gpu
def test_host_resident_labels(host_binary):
    p = subprocess.run([host_binary], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "host_resident_labels_test: all passed" in p.stdout
