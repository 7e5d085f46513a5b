"""CPU model of the snapshot layout without the node_slot fill: gp_build_slots_exec / gp_build_slots_drv decide order
membership from arrays that keep whatever an earlier layout (or a fresh allocation) left in them -- node_slot and the
node -> driver-position scatter drv_pos -- by checking every stale index against what the layout has just rewritten.
Restated in numpy and checked against the rule it replaces (node_slot filled with -1 first) over random stale contents,
including the previous layout's own arrays: driver-only nodes, nodes in neither order, empty groups and orders shorter
than the node table."""
import numpy as np
import pytest


def random_layout(rng, n, n_groups):
    grp = rng.integers(-1, n_groups, n)                       # -1: in neither order
    if n_groups > 2:
        grp[grp == rng.integers(0, n_groups)] = -1            # an empty group
    role = rng.choice(3, n, p=[0.6, 0.2, 0.2])               # 0 both orders, 1 executor only, 2 driver only
    eo, do, eoff, doff = [], [], [0], [0]
    for g in range(n_groups):
        e = rng.permutation(np.nonzero((grp == g) & (role != 2))[0])
        d = rng.permutation(np.nonzero((grp == g) & (role != 1))[0])
        eo += list(e); do += list(d)
        eoff.append(len(eo)); doff.append(len(do))
    return np.array(eo, np.int64), np.array(do, np.int64), np.array(eoff), np.array(doff)


def exec_part(n, eo, eoff, doff, slot_node, node_slot):
    for g in range(len(eoff) - 1):
        sbase = eoff[g] + doff[g]
        for i, v in enumerate(eo[eoff[g]:eoff[g + 1]]):
            slot_node[sbase + i] = v
            node_slot[v] = sbase + i


def driver_part(do, eoff, doff, slot_node, node_slot, drv_slot, genuine):
    for g in range(len(eoff) - 1):
        sbase, ne = eoff[g] + doff[g], eoff[g + 1] - eoff[g]
        for k, v in enumerate(do[doff[g]:doff[g + 1]]):
            j, s = doff[g] + k, sbase + ne + k
            ns = node_slot[v]
            if sbase <= ns < sbase + ne and genuine(ns, v):
                drv_slot[j] = ns - sbase
                slot_node[s] = -1
            else:
                slot_node[s] = v
                node_slot[v] = s
                drv_slot[j] = ne + k


def layout_with_fill(n, eo, do, eoff, doff):
    """the rule the kernels replace: node_slot = -1 everywhere, then the two passes"""
    n_slots = len(eo) + len(do)
    slot_node = np.full(n_slots + 1, -9, np.int64)
    node_slot = np.full(n + 1, -1, np.int64)
    drv_slot = np.full(len(do) + 1, -9, np.int64)
    exec_part(n, eo, eoff, doff, slot_node, node_slot)
    driver_part(do, eoff, doff, slot_node, node_slot, drv_slot, lambda ns, v: True)
    slot_node[n_slots] = -1
    return slot_node, node_slot, drv_slot


def layout_from_stale(n, eo, do, eoff, doff, node_slot, drv_pos, slot_node):
    """the kernels' rule: node_slot, drv_pos and slot_node hold stale values; nothing is filled"""
    n_slots = len(eo) + len(do)
    G = len(eoff) - 1
    used = eoff[G] + doff[G]
    node_slot, drv_pos, slot_node = node_slot.copy(), drv_pos.copy(), slot_node.copy()
    drv_slot = np.full(len(do) + 1, -9, np.int64)
    # K1
    exec_part(n, eo, eoff, doff, slot_node, node_slot)
    for j, v in enumerate(do):
        drv_pos[v] = j
    base = eoff + doff

    def exec_slot(ns, v):                   # an executor slot of its group that K1 gave to v
        g = int(np.searchsorted(base, ns, side="right") - 1)
        return ns - base[g] < eoff[g + 1] - eoff[g] and slot_node[ns] == v

    # K2, node part: -1 for a node in neither order (reads only entries no K2 slot thread writes)
    for v in range(n + 1):
        p = drv_pos[v]
        if 0 <= p < doff[G] and do[p] == v:
            continue
        ns = node_slot[v]
        if not (0 <= ns < used and exec_slot(ns, v)):
            node_slot[v] = -1
    # K2, slot part
    driver_part(do, eoff, doff, slot_node, node_slot, drv_slot, lambda ns, v: slot_node[ns] == v)
    slot_node[used:n_slots + 1] = -1
    return slot_node, node_slot, drv_slot


def stale_arrays(rng, n, n_slots, kind, prev=None):
    if kind == "previous" and prev is not None:
        ns, dp, sn = prev
        fit = lambda a, m: np.resize(a, m) if len(a) else np.full(m, -1, np.int64)
        return fit(ns, n + 1), fit(dp, n + 1), fit(sn, n_slots + 1)
    lo, hi = (-3, max(n, n_slots) + 3) if kind == "near" else (-2**31, 2**31 - 1)
    return (rng.integers(lo, hi, n + 1), rng.integers(lo, hi, n + 1), rng.integers(lo, hi, n_slots + 1))


@pytest.mark.parametrize("seed", range(12))
def test_stale_rule_matches_the_fill(seed):
    rng = np.random.default_rng(seed)
    prev = None
    for _ in range(6):
        n, G = int(rng.integers(1, 300)), int(rng.integers(1, 6))
        eo, do, eoff, doff = random_layout(rng, n, G)
        n_slots = len(eo) + len(do)
        want = layout_with_fill(n, eo, do, eoff, doff)
        for kind in ("near", "wide", "previous"):
            ns, dp, sn = stale_arrays(rng, n, n_slots, kind, prev)
            got = layout_from_stale(n, eo, do, eoff, doff, ns, dp, sn)
            for name, x, y in zip(("slot_node", "node_slot", "drv_slot"), got, want):
                assert np.array_equal(x[:len(y)], y), (seed, kind, name)
        # what this layout leaves behind is the next layout's stale input
        ns0, dp0, sn0 = stale_arrays(rng, n, n_slots, "near")
        sn1, ns1, _ = layout_from_stale(n, eo, do, eoff, doff, ns0, dp0, sn0)
        dp1 = dp0.copy()
        dp1[do] = np.arange(len(do))
        prev = (ns1, dp1, sn1)


def test_order_shorter_than_node_table_and_empty_orders():
    rng = np.random.default_rng(99)
    n = 50
    for eo, do in ((np.array([3, 7], np.int64), np.array([7, 9], np.int64)), (np.array([], np.int64), np.array([1], np.int64)),
                   (np.array([], np.int64), np.array([], np.int64))):
        eoff, doff = np.array([0, len(eo)]), np.array([0, len(do)])
        want = layout_with_fill(n, eo, do, eoff, doff)
        ns, dp, sn = stale_arrays(rng, n, len(eo) + len(do), "near")
        ns[:] = 0; dp[:] = 0                                 # every stale index points at entry 0
        got = layout_from_stale(n, eo, do, eoff, doff, ns, dp, sn)
        for x, y in zip(got, want):
            assert np.array_equal(x[:len(y)], y)
