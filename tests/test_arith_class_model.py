"""The capacity arithmetic's classes and divider kinds, emulated in Python integers (tests/arith_class_model.py), against
floor division over a lattice of requests, numerators and snapshot maxima placed at the class boundaries, and the model
itself pinned to hand-derived recipes of the kernel source."""
import pytest

import arith_class_model as m

ODDS = (3, (1 << 32) - 1, (1 << 32) + 1, (1 << 33) - 1)
QS = (0, 1, 2, (1 << 16) - 1, 1 << 16, 1 << 24, (1 << 32) - 1, 1 << 32)
TS = (0, 1, 2, 8, 16, 28)


def lattice_divisors():
    es = {0, 1}
    es.update(1 << j for j in range(1, 61))
    for o in ODDS:
        j = 0
        while (o << j) < m.MAX_QUANTITY:
            es.add(o << j)
            j += 1
    return sorted(es)


def numerators(e, limit):
    out = {-1}
    for q in QS:
        for d in (-1, 0, 1):
            a = q * max(e, 1) + d
            if 0 <= a < m.MAX_QUANTITY and a <= limit:
                out.add(a)
    return sorted(out)


def maxima():
    return [(1 << (32 + t)) + d for t in TS for d in (-1, 0, 1)]


def test_lattice_every_class_and_kind():
    """For each snapshot maximum M and request e, every class the dispatch allows computes max(0, a // e) for every a in
    [-1, M] of the lattice; the general class is exact for every a."""
    hits = {}
    for e in lattice_divisors():
        for t in (0, 1, 2):
            for mx in maxima():
                dv, fast = m.prep_dim(e, t, mx)
                s = m.shift_for(mx)
                classes = [m.GENERAL]
                if fast:
                    classes.append(m.FAST64)
                    if dv.kind == m.K_MAGIC and s <= dv.sh < s + 32:
                        classes.append(m.FAST32)
                for a in numerators(e, mx):
                    want = m.exact_quotient(a, e)
                    for cls in classes:
                        if cls == m.FAST32 and a > mx:
                            continue
                        got = m.class_quotient(cls, a, dv, s)
                        assert got == want, (cls, m.kind_name(dv), e, t, mx, a, got, want)
                        hits[(cls, m.kind_name(dv))] = hits.get((cls, m.kind_name(dv)), 0) + 1
                # the general path also takes numerators above the maximum (mutable snapshots, reservations)
                for a in numerators(e, m.MAX_QUANTITY):
                    assert m.cap_dim_u(a, dv) == m.exact_quotient(a, e), (e, a)
                    assert m.cap_dim_u(a, m.make_dimdiv(e)) == m.exact_quotient(a, e), (e, a)
    reachable = {(m.GENERAL, k) for k in m.KINDS} | {(c, k) for c in (m.FAST32, m.FAST64) for k in (m.MAGIC2, m.MAGIC)} | \
        {(m.FAST64, m.INF), (m.FAST64, m.SHIFT)}
    assert set(hits) == reachable, sorted(set(hits) ^ reachable)


def test_fast_class_boundary_is_exact():
    """fast is set exactly when max_avail >> sh < 2^32: one below the switch qualifies, the switch itself does not."""
    for sh in (0, 1, 5, 19, 31, 40):
        e = 3 << sh
        assert m.prep_dim(e, 0, ((1 << 32) << sh) - 1)[1]
        assert not m.prep_dim(e, 0, (1 << 32) << sh)[1]
        assert not m.prep_dim(e, 0, ((1 << 32) << sh) + 1)[1]
        # a power of two 2^(sh+1) is prepared as (a >> sh) / 2: the same switch
        assert m.prep_dim(2 << sh, 1, ((1 << 32) << sh) - 1)[1]
        assert not m.prep_dim(2 << sh, 1, (1 << 32) << sh)[1]


def test_shift_for_boundaries():
    assert m.shift_for(-5) == 0 and m.shift_for(0) == 0 and m.shift_for(1) == 0
    assert m.shift_for((1 << 32) - 1) == 0
    for t in range(0, 29):
        assert m.shift_for(1 << (32 + t)) == t + 1
        assert m.shift_for((1 << (32 + t)) - 1) == t
        assert m.shift_for((1 << (32 + t)) + 1) == t + 1
        mx = (1 << (32 + t)) + 1
        assert (mx >> m.shift_for(mx)) < (1 << 32) and (mx >> (m.shift_for(mx) - 1)) >= (1 << 32)


def test_fast64_needs_a_shift_beyond_the_view():
    """A fast application misses the compact view only when a request shift is S + 32 or more (S never exceeds a fast
    request's shift: max >> sh < 2^32 forces sh >= S); such a request exceeds every availability of the snapshot."""
    for mx in maxima():
        s = m.shift_for(mx)
        for e in lattice_divisors():
            dv, fast = m.prep_dim(e, 0, mx)
            if fast and dv.kind == m.K_MAGIC:
                assert dv.sh >= s
                if dv.sh >= s + 32:
                    assert e > mx


def test_hand_derived_recipes():
    """The model against recipes worked out by hand from prep_dim / make_dimdiv / shift_for."""
    g40 = 1 << 40
    assert m.shift_for(g40) == 9
    dv, fast = m.prep_dim(3, 0, g40)
    assert dv == m.DimDiv(0x5555555555555556, 3, 0, m.K_MAGIC) and not fast
    dv, fast = m.prep_dim(3, 0, 64000)
    assert dv == m.DimDiv(0x5555555555555556, 3, 0, m.K_MAGIC) and fast
    dv, fast = m.prep_dim(1 << 20, 1, g40)
    assert dv == m.DimDiv(1 << 63, 1 << 20, 19, m.K_MAGIC) and fast
    assert m.prep_fast32(True, m.prep_dim(1000, 0, 96000)[0], dv, [0, 9])
    dv, fast = m.prep_dim(1, 2, 8)
    assert dv == m.DimDiv(0, 1, 0, m.K_SHIFT) and fast              # gpu: shift allowed in the fast class
    dv, fast = m.prep_dim(1, 0, 8)
    assert dv.kind == m.K_SHIFT and not fast                        # cpu / mem: magic only
    dv, fast = m.prep_dim(0, 1, g40)
    assert dv == m.DimDiv(0, 0, 0, m.K_INF) and not fast            # mem: a zero request leaves the fast class
    assert m.prep_dim(0, 2, g40) == (m.DimDiv(0, 0, 0, m.K_INF), True)
    dv, fast = m.prep_dim(1000, 0, 96000)                           # 1000 = 125 << 3
    assert dv == m.DimDiv(0xFFFFFFFFFFFFFFFF // 125 + 1, 1000, 3, m.K_MAGIC) and dv.magic == 0x20C49BA5E353F7D and fast
    dv, fast = m.prep_dim((1 << 32) + 1, 1, g40)
    assert dv == m.DimDiv(0, (1 << 32) + 1, 0, m.K_SLOW) and not fast
    dv, fast = m.prep_dim(((1 << 32) - 1) << 4, 1, g40)
    assert dv == m.DimDiv(0xFFFFFFFFFFFFFFFF // ((1 << 32) - 1) + 1, ((1 << 32) - 1) << 4, 4, m.K_MAGIC)
    assert dv.magic == 0x100000002 and not fast                     # 2^40 >> 4 = 2^36
    # make_dimdiv: powers of two are shifts, odd parts below 2^32 magic, the rest slow
    assert m.make_dimdiv(0) == m.DimDiv(0, 0, 0, m.K_INF)
    assert m.make_dimdiv(1) == m.DimDiv(0, 1, 0, m.K_SHIFT)
    assert m.make_dimdiv(1 << 30) == m.DimDiv(0, 1 << 30, 30, m.K_SHIFT)
    assert m.make_dimdiv(3 << 30) == m.DimDiv(0x5555555555555556, 3 << 30, 30, m.K_MAGIC)
    assert m.make_dimdiv(((1 << 33) - 1) << 2) == m.DimDiv(0, ((1 << 33) - 1) << 2, 0, m.K_SLOW)
    # fast32: the view's shift has to be at most the request's, and less than 32 below it
    c = m.prep_dim(1000, 0, 96000)[0]
    assert m.prep_fast32(True, c, m.prep_dim(1 << 30, 1, g40)[0], [0, 9])
    assert not m.prep_fast32(True, c, m.prep_dim(1 << 45, 1, g40)[0], [0, 9])      # 44 - 9 = 35 >= 32
    assert not m.prep_fast32(True, m.prep_dim(1 << 34, 0, 96000)[0], m.prep_dim(1 << 30, 1, g40)[0], [0, 9])
    assert not m.prep_fast32(False, c, m.prep_dim(1 << 30, 1, g40)[0], [0, 9])
    # the emulations on worked numbers
    dv = m.prep_dim(3, 0, 64000)[0]
    assert m.fast_q(10, dv) == 3 and m.fast_q(-1, dv) == 0 and m.fast_q(8, dv) == 2
    dv = m.prep_dim(1 << 33, 1, 1 << 60)[0]                         # sh = 32: the funnel shift takes the high word
    assert dv.sh == 32 and m.fast_q((5 << 33) + 7, dv) == 5
    dv = m.prep_dim(3 << 10, 1, g40)[0]
    assert m.cap32_dim(m.compact_pair((7 * 3 << 10) - 1, 9), dv, 9) == 6
    assert m.cap32_dim(m.compact_pair(7 * 3 << 10, 9), dv, 9) == 7
    assert m.compact_pair(-4, 3) == 0 and m.compact_pair((1 << 41) - 1, 9) == (1 << 32) - 1


def test_classify():
    meta = m.SnapMeta([96000, 8000], [(1 << 40) - 1, 1 << 30], [0, 0])
    assert meta.shift32 == [0, 8]
    app = lambda drv, exe: m.App(drv, exe, 1)
    assert m.classify(app((0, 0, 0), (1000, 1 << 30, 0)), meta) == (m.FAST32, (m.MAGIC, m.MAGIC2, m.INF))
    assert m.classify(app((0, 0, 0), (1 << 33, 1 << 30, 0)), meta)[0] == m.FAST64       # cpu sh 32 >= 0 + 32
    assert m.classify(app((0, 0, 0), (1000, 3, 0)), meta)[0] == m.GENERAL                # (2^40 - 1) >> 0 >= 2^32
    assert m.classify(app((0, 0, 1), (1000, 1 << 30, 0)), meta)[0] == m.GENERAL          # gpu binds
    assert m.classify(app((0, 0, 0), (1, 1 << 30, 0)), meta)[0] == m.GENERAL             # cpu e == 1: shift
    neg = m.SnapMeta([96000], [1 << 30], [-1])
    assert m.classify(app((0, 0, 0), (1000, 1 << 30, 0)), neg)[0] == m.GENERAL
    assert m.family_class("fifo", app((0, 0, 1), (1000, 1 << 30, 1)), meta) == m.FAST64
    assert m.family_class("minfrag", app((0, 0, 0), (1 << 33, 1 << 30, 0)), meta) == m.GENERAL


@pytest.mark.parametrize("e", [3, 1000, (1 << 32) - 1, 3 << 20, 1 << 20])
def test_cap32_equals_general_on_every_compact_value(e):
    """Caps<true>::cap32 over compact_pair == cap_dim for numerators at every multiple boundary up to the maximum."""
    for t in (0, 3, 12):
        mx = (1 << (32 + t)) - 1
        dv, fast = m.prep_dim(e, 1, mx)
        s = m.shift_for(mx)
        if not (fast and s <= dv.sh < s + 32):
            continue
        step = max(1, mx // e // 997)
        for q in range(0, mx // e + 2, step):
            for a in (q * e - 1, q * e, q * e + 1):
                if 0 <= a <= mx:
                    assert m.class_quotient(m.FAST32, a, dv, s) == a // e, (e, t, a)
