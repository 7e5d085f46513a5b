"""The context's snapshot state (k8s-spark-scheduler_b200/csrc/gangpack_held.cuh) driven through every layout entry's
transitions, completed and failed after the commit point, with every requirement's outcome after each step
(tests/held_state_test.cpp).  Host-only: the header has no CUDA in it."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-spark-scheduler_b200", "csrc")


def test_held_state_transitions_and_requirements(tmp_path):
    exe = tmp_path / "held_state_test"
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
                           "-o", str(exe), os.path.join(ROOT, "tests", "held_state_test.cpp")])
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "all passed" in p.stdout
