"""Executable statement of the index-shift emission of gp_decide_tables (csrc/gangpack_tables.cuh), on the CPU.

The table kernel also writes, per (shape, group), the driver-free placement prefix P: P[t] is the node that receives the
t-th executor when every node takes its full (clamped) capacity, t < kPlaceLen.  The decision kernel then emits
ExecutorNodes without walking the table: the driver's node d takes cd = cap(d | driver) instead of c0 = cap(d) executors,
so every executor after its run lands delta = c0 - cd places later in P:

    out[t] = P[t < S(d) + cd ? t : t + delta]        t in [0, k)

This checks that formula against the table walk (tests/test_table_walk_model.py, itself checked against the reference's
definition) on random tables, tightly-pack and distribute-evenly (capacities 0/1), and also states how many prefix words
each emission reads -- what the GPU tests compare with gp_last_stats.nodes_scanned."""
import numpy as np
import pytest

from test_table_walk_model import definition, next_above, tab_at, walk

PLACE_LEN = 256          # kPlaceLen


def place_prefix(caps, length=PLACE_LEN):
    """P as the table kernel writes it: node n covers [S(n), min(S(n) + c(n), length))."""
    P = []
    for n, c in enumerate(caps):
        P += [n] * int(c)
        if len(P) >= length:
            break
    return P[:length]


def shift_emission(P, k, a, c0, cd):
    delta = c0 - cd
    return [P[t if t < a + cd else t + delta] for t in range(k)]


def takes_shift_path(k, c0, cd):
    return k != 0 and k - 1 + (c0 - cd) < PLACE_LEN


def walk_probes(caps, k, dpos, cd):
    """Table words the per-thread walk of gp_decide_tables reads (first_host word included), its control flow verbatim."""
    ne = len(caps)
    tab = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    total = int(np.sum(caps))
    pos = int(np.nonzero(caps)[0][0])
    probes = 2
    prev, placed = 0, 0
    nxt = tab_at(tab, pos + 1, ne, total)
    while placed < k and pos < ne:
        nxt2 = tab_at(tab, pos + 2, ne, total)
        probes += 1
        c = cd if pos == dpos else nxt - prev
        if c == 0:
            if nxt >= total:
                break
            p, pr = next_above(tab, pos + 1, ne, total, nxt)
            probes += pr + 1
            pos, prev = p - 1, nxt
            nxt = tab_at(tab, pos + 1, ne, total)
            continue
        placed += min(c, k - placed)
        prev, nxt, pos = nxt, nxt2, pos + 1
    return probes


def emission_probes(caps, k, dpos, c0, cd):
    """Table words read by the emission of one decision (the driver loop's two words per candidate not included)."""
    if k == 0:
        return 0
    return k if takes_shift_path(k, c0, cd) else walk_probes(caps, k, dpos, cd)


@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("seed", range(3))
def test_index_shift_equals_walk(algo, seed):
    rng = np.random.default_rng(100 + seed)
    checked = shifted = 0
    for _ in range(3000):
        ne = int(rng.integers(1, 400))
        hi = 2 if algo == 1 else int(rng.choice([3, 6, 40]))
        caps = rng.integers(0, hi, ne) * (rng.random(ne) < rng.random())
        total = int(caps.sum())
        if total == 0:
            continue
        tab = np.concatenate([[0], np.cumsum(caps)[:-1]])
        dpos = int(rng.integers(0, ne + 2))
        if dpos < ne:
            c0 = int(caps[dpos])
            cd = int(rng.integers(0, c0 + 1))
            a = int(tab[dpos])
        else:                                      # driver-only node: no executor candidate, no shift
            dpos, c0, cd, a = 0x7fffffff, 0, 0, 0
        room = total - (c0 - cd)
        if algo == 1:
            room = min(room, total - 1)           # the tables decide distribute-evenly only with >= k + 1 hosting nodes
        if room <= 0:
            continue
        k = int(rng.integers(1, min(room, PLACE_LEN + 4) + 1))
        want = walk(tab, ne, total, k, dpos, cd, int(np.nonzero(caps)[0][0]))
        assert want == definition(caps, k, dpos, cd)
        checked += 1
        if takes_shift_path(k, c0, cd):
            got = shift_emission(place_prefix(caps), k, a, c0, cd)
            assert got == want, (ne, k, dpos, c0, cd)
            shifted += 1
    assert checked > 1500 and shifted > 1000


def test_shift_indices_stay_inside_the_written_prefix():
    """Feasibility (S(ne) - delta >= k) and the path condition keep every index below min(total, kPlaceLen)."""
    rng = np.random.default_rng(7)
    for _ in range(5000):
        ne = int(rng.integers(1, 300))
        caps = rng.integers(0, 5, ne)
        total = int(caps.sum())
        if total == 0:
            continue
        d = int(rng.integers(0, ne))
        c0 = int(caps[d]); cd = int(rng.integers(0, c0 + 1))
        room = total - (c0 - cd)
        if room <= 0:
            continue
        k = int(rng.integers(1, room + 1))
        if not takes_shift_path(k, c0, cd):
            continue
        a = int(np.sum(caps[:d]))
        top = max(t if t < a + cd else t + c0 - cd for t in range(k))
        assert top < min(total, PLACE_LEN)


def test_probe_model_counts_the_boundary():
    """k - 1 + delta = kPlaceLen - 1 reads k prefix words; one more executor sends the decision down the walk."""
    caps = np.array([0, 3] + [1] * 600)
    assert emission_probes(caps, 255, 1, 3, 1) == walk_probes(caps, 255, 1, 1)        # 255 - 1 + 2 = 256: walk
    assert emission_probes(caps, 254, 1, 3, 1) == 254                                   # 254 - 1 + 2 = 255: shift
    assert emission_probes(caps, 256, 0x7fffffff, 0, 0) == 256
    assert emission_probes(caps, 257, 0x7fffffff, 0, 0) == walk_probes(caps, 257, 0x7fffffff, 0)
