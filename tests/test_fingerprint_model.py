"""tests/fingerprint_ref.py against gp::shape_fingerprint itself, compiled into a small host program, and the premise of every
crafted set the interning tests use (test_gpu_shape_interning.py, test_gpu_exceeds_capacity.py).  If the hash changes, this
fails instead of the GPU tests quietly colliding nothing."""
import os
import subprocess

import numpy as np
import pytest

import fingerprint_ref as fr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-spark-scheduler_b200", "csrc")
MAXQ = fr.MAX_QUANTITY

PROGRAM = r"""
#include "gangpack_kernels.cuh"
#include <cstdio>
int main() {
    long long a, b, c;
    while (std::scanf("%lld %lld %lld", &a, &b, &c) == 3) std::printf("%llu\n", gp::shape_fingerprint(a, b, c));
    return 0;
}
"""


@pytest.fixture(scope="module")
def kernel_fingerprint(tmp_path_factory):
    """-> f(list of (a, b, c) int64 tuples) -> list of gp::shape_fingerprint values, from the header the library builds"""
    from k8s_spark_scheduler_b200 import native
    d = tmp_path_factory.mktemp("fingerprint")
    src, exe = d / "fp.cu", d / "fp"
    src.write_text(PROGRAM)
    subprocess.check_call([native._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I", CSRC,
                           "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])

    def run(tuples):
        signed = lambda v: v - (1 << 64) if v >= 1 << 63 else v          # the chain passes a fingerprint as int64
        text = "".join(f"{signed(a)} {signed(b)} {signed(c)}\n" for a, b, c in tuples)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.split()
        assert len(out) == len(tuples)
        return [int(v) for v in out]
    return run


def crafted_tuples():
    """every (a, b, c) the crafted sets feed to the fingerprint, in the forms the kernels hash them"""
    out = []
    for x, y in fr.executor_pairs():
        out += [x, y]
    for t in fr.driver_pair():
        out.append((t[0] ^ fr.DRIVER_SALT, t[1], t[2]))
    ex, dr, mixed = fr.full_window_sets()
    out += ex + mixed + [(t[0] ^ fr.DRIVER_SALT, t[1], t[2]) for t in dr]
    sets = fr.shape_count_sets()
    out += sets["exec65"] + [(t[0] ^ fr.DRIVER_SALT, t[1], t[2]) for t in sets["drv300"]]
    a, b, c, ga, gc = fr.marker_rows()
    for row, g in ((a, 0), (b, 0), (a, ga), (c, gc)):
        h = fr.fingerprint(row[3], row[4], row[5])
        h2 = fr.fingerprint(h, row[0], row[1])
        out += [(row[3], row[4], row[5]), (h, row[0], row[1]), (h2, row[2], g)]
    return out


def test_restatement_equals_kernel(kernel_fingerprint):
    rng = np.random.default_rng(2)
    tuples = [(1000, 4 << 30, 0)]
    for scale in (1 << 14, 1 << 34, MAXQ):
        tuples += [tuple(int(v) for v in rng.integers(0, scale, 3)) for _ in range(3000)]
    edges = [0, 1, MAXQ - 1, MAXQ - 2, 1 << 32, (1 << 32) - 1]
    tuples += [(a, b, c) for a in edges for b in edges for c in edges]
    tuples += [(-1, 0, 0), (0, -1, 0), (0, 0, -1), (-(1 << 63), (1 << 63) - 1, 7)]     # int64 wrap (the chain's inputs)
    tuples += crafted_tuples()
    assert fr.fingerprint(1000, 4 << 30, 0) == 249919029608841466
    assert kernel_fingerprint(tuples) == [fr.fingerprint(*t) for t in tuples]


def test_solvers():
    rng = np.random.default_rng(3)
    found = 0
    for _ in range(400):
        x = tuple(int(v) for v in rng.integers(0, 1 << 40, 3))
        d = int(rng.integers(0, 3))
        y = fr.collide(x, d, [int(v) for v in rng.integers(0, 1 << 40, 2)])
        yd = fr.collide_driver(x, d, [int(v) for v in rng.integers(0, 1 << 40, 2)])
        for z, f in ((y, fr.fingerprint), (yd, fr.driver_fingerprint)):
            if z is not None:
                found += 1
                assert z != x and all(0 <= v < MAXQ for v in z) and f(*z) == f(*x)
    assert 40 < found < 250                       # about one solution in eight is below 2^61


def test_executor_and_driver_pairs():
    for d, (x, y) in enumerate(fr.executor_pairs()):
        assert fr.fingerprint(*x) == fr.fingerprint(*y) and x != y
        assert y[d] >= fr.HUGE and all(0 <= v < MAXQ for v in y)
        assert all(v < fr.HUGE for i, v in enumerate(y) if i != d)
    xs = [p[0] for p in fr.executor_pairs()]
    assert len({fr.fingerprint(*x) for x in xs}) == 3             # three pairs, not one group of six
    x, y = fr.driver_pair()
    assert fr.driver_fingerprint(*x) == fr.driver_fingerprint(*y) and x != y and y[1] >= fr.HUGE
    assert fr.fingerprint(*x) != fr.fingerprint(*y)                 # the salt matters


def test_full_window_sets():
    ex, dr, mixed = fr.full_window_sets()
    assert fr.window(1020)[-1] == 11 and 0 in fr.window(1020)     # the window wraps past slot 1023
    assert len(set(ex)) == 17 and {fr.home(fr.fingerprint(*t)) for t in ex} == {1020}
    assert len(set(dr)) == 17 and {fr.home(fr.driver_fingerprint(*t)) for t in dr} == {1020}
    assert len({fr.fingerprint(*t) for t in ex}) == 17 and len({fr.driver_fingerprint(*t) for t in dr}) == 17
    assert len(set(mixed)) == 17 and [fr.home(fr.fingerprint(*t)) for t in mixed] == [1020] * 16 + [1023]
    assert 1023 in fr.window(1020)


def test_shape_count_sets():
    s = fr.shape_count_sets()
    for k, f in (("exec65", fr.fingerprint), ("drv300", fr.driver_fingerprint)):
        homes = [fr.home(f(*t)) for t in s[k]]
        assert len(set(homes)) == len(homes) == len(set(s[k]))     # every request sits in its own home slot
    assert s["exec64"] == s["exec65"][:64] and s["drv64"] == s["drv300"][:64] and s["drv65"] == s["drv300"][:65]


def test_marker_rows():
    a, b, c, ga, gc = fr.marker_rows()
    assert fr.marker_fingerprint(a, 0) == fr.marker_fingerprint(b, 0) and a != b
    assert fr.marker_fingerprint(a, ga) == fr.marker_fingerprint(c, gc) and ga != gc
    assert c[:2] == a[:2] and c[3:] == a[3:] and c[2] >= fr.HUGE and b[2] >= fr.HUGE
    assert all(0 <= v < MAXQ for v in b + c)
