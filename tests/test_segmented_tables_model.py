"""Executable statement of the segmented table build of gp_decide_tables (csrc/gangpack_tables.cuh), on the CPU.

The table phase of the one-launch kernel cuts every (shape, instance group) into segments of kTabSeg nodes that run as
separate work items: a segment scans its own capacities, publishes its sum, finds its base by decoupled look-back over the
status words of the earlier segments of the same (shape, group) -- a warp reads 32 of them at a time and stops at the
nearest inclusive word -- and then writes its prefix words S, its part of the placement prefix P, and, for exactly one
segment each, first_host and total.  This model restates the segment mapping (seg_pre), the look-back and the writes line
by line, runs the segments in random interleavings that respect only what the kernel waits for, and checks every word
against the one-pass definition.  (The CUDA kernel itself is checked against the oracles by the -m gpu tests.)"""
import numpy as np
import pytest

PLACE_LEN = 256
MAX_COUNT = 1 << 24
AGG, INC = 1, 2                     # status flags (bits 62-63 of the status word)


def table_clamp(ne):
    by_len = 0xFFFFFFFF // max(ne, 1)
    return min(by_len, MAX_COUNT)


def one_pass(c, slot_node):
    """The definition: S[i] = sum_{n<i} c[n], total, first hosting position (ne: none), P[t] = node of the t-th executor."""
    ne = len(c)
    S = np.zeros(ne, np.int64)
    if ne:
        S[1:] = np.cumsum(c)[:-1]
    total = int(c.sum())
    nz = np.nonzero(c)[0]
    first = int(nz[0]) if nz.size else ne
    P = []
    for i in range(ne):
        if len(P) >= PLACE_LEN:
            break
        P += [int(slot_node[i])] * min(int(c[i]), PLACE_LEN - len(P))
    return S, total, first, P


def segment_prefix(sizes, seg):
    pre = [0]
    for ne in sizes:
        pre.append(pre[-1] + max(1, -(-ne // seg)))
    return pre


def lookback(status, first, idx):
    """One warp's walk; None while a word it needs is still 0 (the kernel spins there)."""
    excl, end = 0, idx
    while True:
        lanes = [end - 1 - lane for lane in range(32)]
        words = [status[j] if j >= first else (INC, 0) for j in lanes]
        if any(w[0] == 0 for w in words):
            return None
        inc = [lane for lane, w in enumerate(words) if w[0] == INC]
        stop = inc[0] if inc else 31
        excl += sum(w[1] for w in words[:stop + 1])
        if inc:
            return excl
        end -= 32


class Segment:
    """One table work item: step() advances it by one of the points where other items can interleave."""

    def __init__(self, c, slot_node, seg, n_seg, seg_len, per_thread, status, st, out):
        self.c, self.slot_node, self.seg, self.n_seg = c, slot_node, seg, n_seg
        self.seg_len, self.per_thread, self.status, self.st, self.out = seg_len, per_thread, status, st, out
        self.state = 0

    def step(self):
        ne = len(self.c)
        lo, hi = self.seg * self.seg_len, min((self.seg + 1) * self.seg_len, ne)
        if self.state == 0:                                  # scan, publish the aggregate (segment 0: inclusive)
            cs = [int(x) for x in self.c[lo:hi]]
            self.seg_total = sum(cs)
            firsts = [lo + j for j, x in enumerate(cs) if x]
            self.first = firsts[0] if firsts else None
            self.status[self.st] = (INC if self.seg == 0 else AGG, self.seg_total)
            self.state = 1
            return True
        if self.state == 1:                                  # look-back, publish the inclusive word
            if self.seg == 0:
                self.base = 0
            else:
                b = lookback(self.status, self.st - self.seg, self.st)
                if b is None:
                    return False
                self.base = b
                self.status[self.st] = (INC, self.base + self.seg_total)
            self.state = 2
            return True
        # writes: S words per thread, P runs of the threads whose base is below PLACE_LEN, first_host, total
        S, P, fh = self.out["S"], self.out["P"], self.out["first_host"]
        run = self.base
        for t0 in range(lo, hi, self.per_thread):
            tbase = run
            vals = [int(x) for x in self.c[t0:min(t0 + self.per_thread, hi)]]
            acc = 0
            for j, x in enumerate(vals):
                S[t0 + j] = tbase + acc
                if tbase < PLACE_LEN:
                    for t in range(tbase + acc, min(tbase + acc + x, PLACE_LEN)):
                        P[t] = int(self.slot_node[t0 + j])
                acc += x
            run += acc
        if self.base == 0 and self.seg_total != 0:
            fh.append(self.first)
        if self.seg == self.n_seg - 1:
            self.out["total"].append(self.base + self.seg_total)
            if self.base + self.seg_total == 0:
                fh.append(ne)
        self.state = 3
        return True


def build_segmented(rng, caps_by_group, slots_by_group, seg_len, per_thread):
    """Every group of one shape, the segments as work items in ticket order, run in a random interleaving: an item can
    only be stuck on items with smaller tickets."""
    pre = segment_prefix([len(c) for c in caps_by_group], seg_len)
    status = [(0, 0)] * pre[-1]
    outs, items = [], []
    for g, (c, sn) in enumerate(zip(caps_by_group, slots_by_group)):
        out = {"S": [None] * len(c), "P": [None] * PLACE_LEN, "first_host": [], "total": []}
        outs.append(out)
        n_seg = pre[g + 1] - pre[g]
        items += [Segment(c, sn, s, n_seg, seg_len, per_thread, status, pre[g] + s, out) for s in range(n_seg)]
    live = list(range(len(items)))
    while live:
        k = int(rng.integers(0, min(len(live), 6)))          # one of the few oldest claimed tickets moves on
        if not items[live[k]].step():
            k = 0                                            # stuck on a smaller ticket; the oldest one never is
            assert items[live[0]].step(), "the oldest claimed ticket waits"
        if items[live[k]].state == 3:
            live.pop(k)
    return outs


def clamp_caps(raw, algo):
    c = np.minimum(raw, table_clamp(len(raw))).astype(np.int64)
    return (c != 0).astype(np.int64) if algo == 1 else c


@pytest.mark.parametrize("seed", range(12))
def test_segmented_build_equals_one_pass(seed):
    rng = np.random.default_rng(seed)
    seg_len = int(rng.choice([8, 32, 64, 1024]))
    per_thread = int(rng.choice([1, 4])) if seg_len >= 8 else 1
    sizes = [0, 1, seg_len - 1, seg_len, seg_len + 1, 3 * seg_len + int(rng.integers(0, seg_len)),
             (40 if seg_len <= 64 else 2) * seg_len + 3, int(rng.integers(0, 5 * seg_len))]   # > 32 segments: several windows
    sizes = [sizes[i] for i in rng.permutation(len(sizes))]
    algo = seed % 2
    caps, slots = [], []
    base = 0
    for ne in sizes:
        raw = rng.integers(0, 5, ne) * (rng.random(ne) < rng.random())
        if rng.random() < 0.3:                              # counts around the clamp
            raw = np.where(rng.random(ne) < 0.01, rng.integers(1 << 23, 1 << 26, ne), raw)
        caps.append(clamp_caps(raw, algo))
        slots.append(np.arange(base, base + ne) * 7 + 3)
        base += ne
    outs = build_segmented(rng, caps, slots, seg_len, per_thread)
    for c, sn, out in zip(caps, slots, outs):
        S, total, first, P = one_pass(c, sn)
        assert out["S"] == [int(x) for x in S]
        assert out["total"] == [total]
        assert out["first_host"] == [first]                 # written by exactly one segment
        assert out["P"][:len(P)] == P
        assert all(x is None for x in out["P"][len(P):])    # entries t >= total are not written
        assert total <= 0xFFFFFFFF                          # the uint32 words do not wrap under the clamp


def test_segment_prefix_counts_empty_groups():
    assert segment_prefix([0, 1, 1023, 1024, 1025, 0], 1024) == [0, 1, 2, 3, 4, 6, 7]
    # the bound the host sizes the status words by: sum max(1, ceil(ne / seg)) <= n_slots / seg + n_groups
    rng = np.random.default_rng(1)
    for _ in range(200):
        sizes = rng.integers(0, 5000, int(rng.integers(1, 400)))
        assert segment_prefix(sizes, 1024)[-1] <= int(sizes.sum()) // 1024 + len(sizes)


def test_lookback_windows():
    """Chains longer than one warp's window: aggregates are summed window by window until an inclusive word."""
    rng = np.random.default_rng(2)
    for n in (1, 2, 31, 32, 33, 64, 65, 200):
        vals = rng.integers(0, 1000, n)
        for inc_at in (0, n // 2, n - 1):
            status = [(AGG, int(v)) for v in vals]
            status[0] = (INC, int(vals[0]))
            status[inc_at] = (INC, int(vals[:inc_at + 1].sum()))
            for idx in range(1, n):
                assert lookback(status, 0, idx) == int(vals[:idx].sum())
        status = [(AGG, int(v)) for v in vals]
        status[0] = (0, 0)
        if n > 1:
            assert lookback(status, 0, n - 1) is None      # still waiting for the first segment
