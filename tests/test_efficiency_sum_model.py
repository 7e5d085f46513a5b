"""CPU model of the exact accumulator of gp_packing_efficiency (csrc/gangpack_efficiency.cuh).

The device sums the reference's per-node packing-efficiency terms in a 256-bit two's-complement fixed-point integer with
its least significant bit at 2^-113 (four 64-bit limbs, add with carry) and rounds the total once, to nearest-even.  This
file restates the conversion, the limb arithmetic and the rounding step by step as the kernels do them and checks them
against fractions.Fraction-exact rounding and math.fsum on adversarial sets, the row update (base minus unreserved plus
reserved) against a from-scratch sum, and the range bound the kernel comment states against the reference's terms.
"""
import math
import os
import random
import struct
import sys
from fractions import Fraction

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import pyref  # noqa: E402

FRAC = 113
M64 = (1 << 64) - 1


# ---- the device model, limb by limb ---------------------------------------------------------------------------------
def fx_zero():
    return [0, 0, 0, 0]


def fx_add(a, b):
    """fx_add: four 64-bit adds with carry."""
    out, carry = [], 0
    for i in range(4):
        s = (a[i] + b[i]) & M64
        c1 = 1 if s < a[i] else 0
        t = (s + carry) & M64
        c2 = 1 if t < s else 0
        out.append(t)
        carry = c1 | c2
    return out


def fx_neg(a):
    out, carry = [], 1
    for i in range(4):
        t = ((~a[i]) + carry) & M64
        carry = 1 if (carry and t == 0) else 0
        out.append(t)
    return out


def fx_from_double(x):
    """fx_add_double's conversion: None when x is not a multiple of 2^-113 below 2^192 (the kernel's range error)."""
    if x == 0.0:
        return fx_zero()
    bits = struct.unpack("<Q", struct.pack("<d", x))[0]
    ex = (bits >> 52) & 0x7FF
    m = bits & ((1 << 52) - 1)
    if ex == 0:
        e = -1074
    else:
        m |= 1 << 52
        e = ex - 1075
    s = e + FRAC
    if s < 0:                                       # trailing zero bits below 2^-113 may be dropped, nothing else
        if s <= -53 or m & ((1 << -s) - 1):
            return None
        m >>= -s
        s = 0
    if s > 192 - 53:
        return None
    li, off = s >> 6, s & 63
    lo, hi = (m << off) & M64, (m >> (64 - off)) if off else 0
    v = [0, 0, 0, 0]
    v[li] = lo
    v[li + 1] = hi
    return fx_neg(v) if bits >> 63 else v


def fx_any_below(a, p):
    for i in range(4):
        r = p - 64 * i
        mask = M64 if r >= 64 else ((1 << r) - 1 if r > 0 else 0)
        if a[i] & mask:
            return True
    return False


def fx_bits_at(a, p):
    li, off = p >> 6, p & 63
    limb = lambda i: a[i] if 0 <= i < 4 else 0
    v = limb(li) >> off
    if off:
        v |= (limb(li + 1) << (64 - off)) & M64
    return v


def fx_to_double(a):
    """fx_to_double: round-to-nearest-even of a * 2^-113; zero is +0.0."""
    neg = a[3] >> 63 == 1
    if neg:
        a = fx_neg(a)
    top = 3 if a[3] else 2 if a[2] else 1 if a[1] else 0 if a[0] else -1
    if top < 0:
        return 0.0
    h = 64 * top + a[top].bit_length() - 1
    if h <= 52:
        r = math.ldexp(float(a[0]), -FRAC)
    else:
        shift = h - 52
        m = fx_bits_at(a, shift) & ((1 << 53) - 1)
        half = fx_bits_at(a, shift - 1) & 1
        sticky = fx_any_below(a, shift - 1)
        if half and (sticky or (m & 1)):
            m += 1
            if m == 1 << 53:
                m >>= 1
                shift += 1
        r = math.ldexp(float(m), shift - FRAC)
    return -r if neg else r


def device_sum(terms):
    acc = fx_zero()
    for t in terms:
        v = fx_from_double(t)
        assert v is not None, t
        acc = fx_add(acc, v)
    return fx_to_double(acc)


def exact_round(terms):
    """Fraction-exact sum rounded once to nearest-even (int / int true division is correctly rounded)."""
    f = sum((Fraction(t) for t in terms), Fraction(0))
    return f.numerator / f.denominator


def check(terms):
    got = device_sum(terms)
    want = exact_round(terms)
    assert got == want and math.copysign(1.0, got) == math.copysign(1.0, want), (got, want)
    fs = math.fsum(terms)
    assert got == fs, (got, fs)
    return got


def pow2_range_terms(rng, n):
    return [rng.choice((1, -1)) * math.ldexp(rng.getrandbits(53) | (1 << 52), rng.randint(-61, 62) - 52) for _ in range(n)]


# ---- the adversarial sets ---------------------------------------------------------------------------------------------
def test_terms_from_2m61_to_2p62():
    rng = random.Random(1)
    check([math.ldexp(1.0, e) for e in range(-61, 63)])
    check([-math.ldexp(1.0, e) for e in range(-61, 63)])
    for _ in range(200):
        check(pow2_range_terms(rng, rng.randint(1, 60)))


def test_extremes_of_the_range():
    check([math.ldexp(1.0, -61)])
    check([math.ldexp(1.0, 63)] * 5 + [math.ldexp(1.0, -61)])
    check([math.ldexp((1 << 53) - 1, 63 - 53)] * 3 + [-math.ldexp(1.0, -61)])
    # below 2^-113 granularity the conversion refuses (the kernel's range error), it never truncates
    assert fx_from_double(math.ldexp(1.0, -114)) is None
    assert fx_from_double(math.ldexp(1.0, -113)) == [1, 0, 0, 0]
    assert fx_from_double(math.ldexp(3.0, -113)) == [3, 0, 0, 0]
    assert fx_from_double(math.ldexp(1.0 + 2.0 ** -52, -70)) is None
    assert fx_from_double(math.ldexp(1.0, 193)) is None
    # beyond the terms' domain but inside the accumulator: the 53 bits start in limb 2 (s >= 128) and are placed exactly
    assert fx_from_double(math.ldexp(1.0, 70)) == [0, 0, 1 << (70 + FRAC - 128), 0]
    assert fx_from_double(math.ldexp(1.0, 15)) == [0, 0, 1, 0]                    # 2^15 = 2^128 units: bit 0 of limb 2
    assert fx_from_double(math.ldexp(1.0, 14)) == [0, 1 << 63, 0, 0]
    for e in (15, 64, 67, 70, 78):
        x = math.ldexp((1 << 53) - 1, e - 52)
        assert fx_to_double(fx_from_double(x)) == x and fx_to_double(fx_from_double(-x)) == -x
        check([x, math.ldexp(1.0, -61), -x])
        check([x, 3.0, math.ldexp(1.0, -61)])
    assert fx_from_double(math.ldexp((1 << 53) - 1, 78 - 52)) == [0, 0, ((1 << 53) - 1) << 11, 0]   # top bit = bit 191
    assert fx_from_double(math.ldexp(1.0, 79)) is None              # the first power of two whose top bit would pass bit 191


def test_massive_cancellation():
    rng = random.Random(2)
    for _ in range(200):
        tiny = pow2_range_terms(rng, rng.randint(1, 8))
        tiny = [math.ldexp(abs(t), -rng.randint(0, 60)) if abs(t) > 1 else t for t in tiny]
        big = []
        for _ in range(rng.randint(1, 10)):
            v = math.ldexp(rng.getrandbits(53) | (1 << 52), 62 - 52)
            big += [v, -v]
        terms = big + tiny
        rng.shuffle(terms)
        check(terms)
    # a left-to-right float64 loop (the Go sum) loses the tiny term entirely
    terms = [math.ldexp(1.0, 62), math.ldexp(1.0, -61), -math.ldexp(1.0, 62)]
    naive = 0.0
    for t in terms:
        naive += t
    assert naive == 0.0
    assert check(terms) == math.ldexp(1.0, -61)


def test_half_ulp_ties():
    one = 1.0
    half_ulp = math.ldexp(1.0, -53)
    assert check([one, half_ulp]) == 1.0                                   # tie -> even (1.0)
    odd = 1.0 + math.ldexp(1.0, -52)
    assert check([odd, half_ulp]) == odd + math.ldexp(1.0, -52)           # tie -> even (up)
    assert check([one, half_ulp, math.ldexp(1.0, -61)]) == 1.0 + math.ldexp(1.0, -52)   # sticky bit breaks the tie
    assert check([-odd, -half_ulp]) == -(odd + math.ldexp(1.0, -52))
    big = math.ldexp(1.0, 62)
    assert check([big, math.ldexp(1.0, 62 - 53)]) == big
    rng = random.Random(3)
    for _ in range(300):
        base = math.ldexp(rng.getrandbits(53) | (1 << 52), rng.randint(-60, 9))
        ulp = math.ulp(base)
        check([base, ulp / 2])
        check([base, -ulp / 2])
        check([base, ulp / 2, math.ldexp(ulp, -40)])
    # carry out of the 53-bit mantissa on rounding up: (2^53 - 1) + 1/2 -> 2^53
    assert check([float((1 << 53) - 1), 0.5]) == float(1 << 53)


def test_zero_and_negative_zero():
    for terms in ([], [0.0], [-0.0], [-0.0, -0.0], [0.0, -0.0, 0.0], [1.5, -1.5], [-2.0, 2.0, -0.0]):
        got = device_sum(terms)
        assert got == 0.0 and math.copysign(1.0, got) == 1.0, terms
        assert got == exact_round(terms)


def test_limb_carry_chains():
    # carries that ripple across every limb, and borrows back
    a = [M64, M64, M64, 0]
    assert fx_add(a, [1, 0, 0, 0]) == [0, 0, 0, 1]
    assert fx_add([0, 0, 0, 1], fx_neg([1, 0, 0, 0])) == [M64, M64, M64, 0]
    assert fx_neg(fx_zero()) == fx_zero()
    rng = random.Random(4)
    for _ in range(2000):
        x = rng.getrandbits(250) * rng.choice((1, -1))
        y = rng.getrandbits(250) * rng.choice((1, -1))
        to = lambda v: [(v % (1 << 256)) >> (64 * i) & M64 for i in range(4)]
        assert fx_add(to(x), to(y)) == to(x + y)
        assert fx_neg(to(x)) == to(-x)


def test_2p20_random_terms():
    rng = random.Random(5)
    n = 1 << 20
    terms = [rng.choice((1, -1)) * math.ldexp(rng.getrandbits(53), rng.randint(-60, 40) - 52) for _ in range(n)]
    got = device_sum(terms)
    assert got == math.fsum(terms)
    assert got == exact_round(terms)


# ---- the row update: base minus unreserved plus reserved --------------------------------------------------------------
def _cluster(rng, n):
    nodes = []
    for _ in range(n):
        sc = rng.choice((0, -1000, rng.randint(1, 64_000), rng.randint(1, 64) * 1000 + rng.randint(0, 999)))
        sm = rng.choice((0, -(1 << 30), rng.randint(1, 1 << 40)))
        sg = rng.choice((0, 0, 0, 8, -1))
        ac = sc - rng.randint(-20_000, max(sc, 1))
        am = sm - rng.randint(-(1 << 32), max(sm, 1))
        ag = sg - rng.randint(-2, 8)
        nodes.append(((ac, am, ag), (sc, sm, sg)))
    return nodes


def _terms(nodes, reserved):
    cpu, mem, gpu, mx = [], [], [], []
    for i, (av, sc) in enumerate(nodes):
        c, m, g = pyref.compute_packing_efficiency(av, sc, reserved.get(i))
        cpu.append(c); mem.append(m); mx.append(max(g, max(c, m)))
        if sc[2] != 0:
            gpu.append(g)
    return cpu, mem, gpu, mx


def test_row_update_equals_from_scratch():
    rng = random.Random(6)
    for trial in range(60):
        nodes = _cluster(rng, rng.randint(1, 60))
        base = [fx_zero() for _ in range(4)]
        for j, col in enumerate(_terms(nodes, {})):
            for t in col:
                base[j] = fx_add(base[j], fx_from_double(t))
        for _ in range(5):
            d = rng.randrange(len(nodes))
            ex = [rng.randrange(len(nodes)) for _ in range(rng.randint(0, 12))]
            drv, exe = (rng.randint(0, 9000), rng.randint(0, 1 << 34), rng.randint(0, 2)), (rng.randint(0, 9000), rng.randint(0, 1 << 34), 1)
            reserved = pyref._reserved_of(drv, exe, d, ex) if trial % 3 else {d: drv}
            acc = [list(b) for b in base]
            for n in sorted(set([d] + ex)):
                av, sc = nodes[n]
                c0, m0, g0 = pyref.compute_packing_efficiency(av, sc, None)
                c1, m1, g1 = pyref.compute_packing_efficiency(av, sc, reserved.get(n))
                olds = (c0, m0, g0, max(g0, max(c0, m0)))
                news = (c1, m1, g1, max(g1, max(c1, m1)))
                for j in range(4):
                    if j == 2 and sc[2] == 0:
                        continue
                    acc[j] = fx_add(acc[j], fx_from_double(-olds[j]))
                    acc[j] = fx_add(acc[j], fx_from_double(news[j]))
            scratch = _terms(nodes, reserved)
            for j in range(4):
                got = fx_to_double(acc[j])
                assert got == math.fsum(scratch[j]) == exact_round(scratch[j]), (trial, j)


def test_term_range_bound_against_reference_terms():
    """The bound of the kernel comment: with |sched|, |avail| < 2^61 and reserved + add-back < 2^61 every term is a multiple
    of 2^-113 and at most 2^63 in magnitude, so it converts without loss."""
    rng = random.Random(7)
    lim = (1 << 61) - 1
    edge = (0, 1, -1, 999, 1000, 1001, lim, -lim, lim - 1, 1 << 40)
    for _ in range(20000):
        pick = lambda: rng.choice(edge) if rng.random() < 0.5 else rng.randint(-lim, lim)
        sc = (pick(), pick(), pick())
        av = (pick(), pick(), pick())
        res = tuple(rng.choice((0, lim, rng.randint(0, lim))) for _ in range(3))
        for t in pyref.compute_packing_efficiency(av, sc, res):
            assert abs(t) <= 2.0 ** 63
            assert t == 0.0 or abs(t) >= 2.0 ** -61
            assert fx_from_double(t) is not None
            assert Fraction(t) * (1 << FRAC) == int(Fraction(t) * (1 << FRAC))
