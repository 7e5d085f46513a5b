"""gp_pack_fifo_zones_groups: fitEarlierDrivers (resource.go:224-262) of every instance group at once with a zone-aware
packer, one CTA per instance group.  For every instance group the outputs must be what gp_pack_fifo_zones /
gp_pack_fifo_az_aware return on a context that holds only that instance group's groups and applications, and what the
literal restatement's loop (orc_fifo) returns over that instance group's node orders: driver_node (-1 / -2 included), the
local zone, every ExecutorNodes slice, the averages as uint64 bits, the availability left behind and the summed gp_stats."""
import numpy as np
import pytest

from helpers import node_names, random_apps, random_cluster, res_aos

pytestmark = pytest.mark.gpu

SINGLE_TIGHT, SINGLE_MINFRAG, AZ_AWARE = 3, 4, 2                  # gp_binpacker
ORC_ALGO = {SINGLE_TIGHT: 2, SINGLE_MINFRAG: 5, AZ_AWARE: 3}       # the literal oracle's packer ids
PACKERS = [SINGLE_TIGHT, SINGLE_MINFRAG, AZ_AWARE]


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


@pytest.fixture(scope="module")
def alone(gangpack):
    """a second context: one instance group at a time through the single-group entry points"""
    p = gangpack.GangPacker()
    yield p
    p.close()


def zone_layout(order_d, order_e, zone_of, az):
    """One instance group's snapshot groups: its candidate zones in driverZonesInOrder order (zones without executor
    candidates left out, single_az.go:36-41) holding the orders restricted to them; az-aware adds one trailing group with
    every other node of the two orders.  -> (n_zones, exec_order, drv_order, exec_off, drv_off)."""
    zones, dz, ez = [], {}, {}
    for n in order_d:
        z = zone_of[n]
        if z not in dz:
            zones.append(z); dz[z] = []
        dz[z].append(n)
    for n in order_e:
        ez.setdefault(zone_of[n], []).append(n)
    zones = [z for z in zones if z in ez]
    eoff, doff, eo, do = [0], [0], [], []
    for z in zones:
        eo += ez[z]; do += dz[z]
        eoff.append(len(eo)); doff.append(len(do))
    if az:
        cand = set(zones)
        te = [n for n in order_e if zone_of[n] not in cand]
        td = [n for n in order_d if zone_of[n] not in cand]
        if te or td or not zones:
            eo += te; do += td
            eoff.append(len(eo)); doff.append(len(do))
    return len(zones), eo, do, eoff, doff


class Case:
    """A cluster of instance groups: node indices interleaved over the groups, per group its zones and node orders."""

    def __init__(self, rng, zones_per_group, per_zone=3, gpus=False, no_zone=()):
        self.G = len(zones_per_group)
        sizes = [max(z, 2) * per_zone + 2 for z in zones_per_group]
        self.n = n = int(sum(sizes))
        owner = rng.permutation(np.repeat(np.arange(self.G), sizes))
        self.cpu, self.mem, self.gpu = random_cluster(rng, n, gpus=gpus)
        self.sc = self.cpu + rng.integers(0, 9, n) * 250 + (rng.integers(0, 3, n) == 0) * 1
        self.sm = self.mem + rng.integers(0, 17, n) * (1 << 28)
        self.sg = np.maximum(self.gpu, 0) + (rng.integers(0, 2, n) if gpus else 0)
        self.zone_of = np.zeros(n, np.int64)
        self.orders, self.exec_only = [], []
        for i, Z in enumerate(zones_per_group):
            nodes = np.nonzero(owner == i)[0]
            self.exec_only.append(int(nodes[-1]))
            if i in no_zone:                      # drivers only in zone 0, executors only in zone 1: no candidate zone
                self.zone_of[nodes] = np.arange(len(nodes)) % 2
                order_d = [int(v) for v in rng.permutation(nodes) if self.zone_of[v] == 0]
                order_e = [int(v) for v in rng.permutation(nodes) if self.zone_of[v] == 1]
            else:
                # zones 0..Z-1 hold both kinds of candidates; two extra nodes: a driver-only and an executor-only zone
                self.zone_of[nodes[:-2]] = rng.permutation(np.arange(len(nodes) - 2) % Z)
                self.zone_of[nodes[-2]], self.zone_of[nodes[-1]] = Z, Z + 1
                first = {}
                for v in nodes[:-2]:
                    first.setdefault(int(self.zone_of[v]), int(v))
                keep = set(first.values())
                order_e = [int(v) for v in rng.permutation(nodes) if v != nodes[-2]]
                order_d = [int(v) for v in rng.permutation(nodes) if v != nodes[-1] and (v in keep or rng.random() < 0.7)]
            self.orders.append((order_d, order_e))
        self.names = node_names(n)
        self.labels = ["g%d-z%d" % (int(owner[v]), int(self.zone_of[v])) for v in range(n)]

    def layout(self, az):
        """-> (snapshot exec_order, drv_order, exec_off, drv_off, group_off, n_zones, undivided exec_off, exec_order,
        drv_off, drv_order), and per instance group its own (n_zones, exec_order, drv_order, exec_off, drv_off)"""
        eo, do, eoff, doff, goff, nz, per = [], [], [0], [0], [0], [], []
        for order_d, order_e in self.orders:
            z, e, d, eo_i, do_i = zone_layout(order_d, order_e, self.zone_of, az)
            per.append((z, e, d, eo_i, do_i))
            eoff += [len(eo) + x for x in eo_i[1:]]; doff += [len(do) + x for x in do_i[1:]]
            eo += e; do += d
            goff.append(goff[-1] + len(eo_i) - 1); nz.append(z)
        uo_e = [v for _, e in self.orders for v in e]
        uo_d = [v for d, _ in self.orders for v in d]
        ue_off = np.cumsum([0] + [len(e) for _, e in self.orders]); ud_off = np.cumsum([0] + [len(d) for d, _ in self.orders])
        i32 = lambda x: np.array(x, np.int32)
        snap = (i32(eo), i32(do), i32(eoff), i32(doff))
        kw = dict(group_off=i32(goff))
        if az:
            kw.update(n_zones=i32(nz), exec_off=i32(ue_off), exec_order=i32(uo_e), drv_off=i32(ud_off), drv_order=i32(uo_d))
        return snap, kw, per

    def load(self, p, az):
        snap, kw, per = self.layout(az)
        p.set_snapshot(self.cpu, self.mem, self.gpu, *snap)
        p.set_schedulable(self.sc, self.sm, self.sg)
        return kw, per


def make_apps(rng, G, q, gpus=False, skip_groups=(), big=0.12):
    apps = random_apps(rng, q, gpus=gpus)
    apps["count"] = np.where(rng.random(q) < big, rng.integers(15, 60, q), apps["count"]).astype(np.int32)
    apps["young"] = (rng.random(q) < 0.97).astype(np.uint8)
    live = [g for g in range(G) if g not in skip_groups]
    apps["group"] = rng.choice(live, size=q).astype(np.int32)           # instance groups interleaved in queue order
    return apps


def subset(apps, sel):
    return {k: np.asarray(v)[sel] for k, v in apps.items()}


def run_groups(p, case, apps, packer_id, mode):
    az = packer_id == AZ_AWARE
    kw, per = case.load(p, az)
    out = p.pack_fifo_zones_groups(apps, packer_id, mode, **kw)
    return out, p.get_snapshot(), p.stats(), per


def expected(case, alone, oracle, apps, packer_id, mode, per):
    """Per instance group: the single-group entry on a context holding only its groups, and the literal loop over its
    orders.  -> per-application (zone, driver, ExecutorNodes list, avg), final availability, summed stats."""
    az = packer_id == AZ_AWARE
    q = len(apps["count"])
    zone = np.full(q, -9, np.int32); drv = np.full(q, -9, np.int32); avg = np.zeros((q, 4)); exe = [None] * q
    avail = [a.copy() for a in (case.cpu, case.mem, case.gpu)]
    stats = {"nodes_scanned": 0, "drivers_tried": 0, "scan_path_apps": 0}
    cl = oracle.Cluster(case.names, case.cpu, case.mem, case.gpu, sched=(case.sc, case.sm, case.sg), zone=case.labels)
    for i, (order_d, order_e) in enumerate(case.orders):
        sel = np.nonzero(apps["group"] == i)[0]
        if sel.size == 0:
            continue
        sub = subset(apps, sel)
        drv_r = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"]); exe_r = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
        _, wd, we, woff = cl.fifo(ORC_ALGO[packer_id], mode, drv_r, exe_r, sub["count"], sub["young"],
                                  [case.names[v] for v in order_d], [case.names[v] for v in order_e])
        z_i, e_i, d_i, eoff_i, doff_i = per[i]
        if len(eoff_i) == 1:                  # single-AZ without a candidate zone: EmptyPackingResult for everyone
            gz = np.full(len(sel), -1, np.int32); gd = wd; goff = woff; ge = we; gavg = np.zeros((len(sel), 4))
            assert (wd < 0).all()
        else:
            alone.set_snapshot(case.cpu, case.mem, case.gpu, np.array(e_i, np.int32), np.array(d_i, np.int32),
                               np.array(eoff_i, np.int32), np.array(doff_i, np.int32))
            alone.set_schedulable(case.sc, case.sm, case.sg)
            if az:
                gz, gd, ge, goff, gavg = alone.pack_fifo_az_aware(sub, mode, order_e, order_d, z_i)
            else:
                gz, gd, ge, goff, gavg = alone.pack_fifo_zones(sub, 0 if packer_id == SINGLE_TIGHT else 2, mode)
            st = alone.stats()
            for k in stats:
                stats[k] += st[k]
            snap = alone.get_snapshot()
            nodes = np.array(sorted(set(order_d) | set(order_e)), np.int64)
            for a, s in zip(avail, snap):
                a[nodes] = s[nodes]
            assert np.array_equal(gd, wd), (i, np.nonzero(gd != wd)[0][:5])
            for j in np.nonzero(wd >= 0)[0]:
                assert np.array_equal(ge[goff[j]:goff[j + 1]], we[woff[j]:woff[j + 1]]), (i, j)
        for j, a in enumerate(sel):
            zone[a], drv[a], avg[a] = gz[j], gd[j], gavg[j]
            exe[a] = list(ge[goff[j]:goff[j + 1]]) if gd[j] >= 0 else None
    for x, y in zip(avail, cl.available()):
        assert np.array_equal(x, y)
    return zone, drv, exe, avg, avail, stats


def check(case, packer, alone, oracle, apps, packer_id, mode, label):
    (zone, drv, ge, goff, avg), snap, st, per = run_groups(packer, case, apps, packer_id, mode)
    wz, wd, we, wavg, wavail, wst = expected(case, alone, oracle, apps, packer_id, mode, per)
    bad = np.nonzero(drv != wd)[0]
    assert bad.size == 0, (label, bad[:5], drv[bad[:5]], wd[bad[:5]])
    assert np.array_equal(zone, wz), (label, np.nonzero(zone != wz)[0][:5])
    for j in np.nonzero(wd >= 0)[0]:
        assert list(ge[goff[j]:goff[j + 1]]) == we[j], (label, j)
    assert np.array_equal(avg.view(np.uint64), wavg.view(np.uint64)), label
    for x, y in zip(snap, wavail):
        assert np.array_equal(x, y), label
    for k in wst:
        assert st[k] == wst[k], (label, k, st[k], wst[k])
    return zone, drv, st


@pytest.mark.parametrize("packer_id", PACKERS)
@pytest.mark.parametrize("G", [1, 2, 7, 140])
def test_random_instance_groups_vs_oracle(oracle, packer, alone, packer_id, G):
    rng = np.random.default_rng(9100 + 10 * G + packer_id)
    zones = [int(z) for z in rng.integers(1, 5, G)]
    case = Case(rng, zones, gpus=G == 7)
    apps = make_apps(rng, G, 40 * G if G < 140 else 1400, gpus=G == 7)
    for mode in (1, 2):
        zone, drv, st = check(case, packer, alone, oracle, apps, packer_id, mode, f"G={G} packer={packer_id} mode={mode}")
        assert (drv >= 0).any()
        if packer_id == AZ_AWARE and G >= 7:
            assert st["scan_path_apps"] > 0                             # the fallback ran


@pytest.mark.parametrize("packer_id", PACKERS)
def test_zone_counts_and_an_idle_group(oracle, packer, alone, packer_id):
    """Instance groups with 1, 17 (more zones than the CTA's 16 warps) and 64 zones, one without a candidate zone
    (single-AZ: EmptyPackingResult and blocking; az-aware: plain tightly-pack over its trailing group) and one without
    applications."""
    rng = np.random.default_rng(9300 + packer_id)
    zones = [1, 17, 64, 2, 3, 2]
    case = Case(rng, zones, no_zone=(3,))
    apps = make_apps(rng, len(zones), 700, skip_groups=(5,))
    for mode in (1, 2):
        zone, drv, st = check(case, packer, alone, oracle, apps, packer_id, mode, f"zones packer={packer_id} mode={mode}")
        g3 = apps["group"] == 3
        if packer_id == AZ_AWARE:
            assert (zone[g3] == -1).all() and (drv[g3] >= 0).any()
        else:
            assert (drv[g3] < 0).all()
        assert (zone[apps["group"] == 2] >= 16).any()                   # a zone of the second warp stride won


@pytest.mark.parametrize("packer_id", PACKERS)
def test_gpu_bound_groups(oracle, packer, alone, packer_id):
    rng = np.random.default_rng(9400 + packer_id)
    case = Case(rng, [3, 4, 2, 3], gpus=True)
    apps = make_apps(rng, 4, 300, gpus=True)
    apps["exe_gpu"] = np.maximum(apps["exe_gpu"], 1)                    # every executor needs a gpu
    for mode in (1, 2):
        check(case, packer, alone, oracle, apps, packer_id, mode, f"gpu packer={packer_id} mode={mode}")


@pytest.mark.parametrize("packer_id", PACKERS)
def test_a_blocked_queue_blocks_its_own_group_only(oracle, packer, alone, packer_id):
    rng = np.random.default_rng(9500 + packer_id)
    case = Case(rng, [3, 2, 4])
    apps = make_apps(rng, 3, 240)
    a = np.nonzero(apps["group"] == 1)[0]
    others = apps["group"] != 1
    apps["drv_cpu"][a[0]] = 1 << 40                                     # group 1's first driver fits nowhere ...
    apps["young"][a[0]] = 0                                             # ... and is not young
    without = subset(apps, others)
    for mode in (1, 2):
        zone, drv, _ = check(case, packer, alone, oracle, apps, packer_id, mode, f"blocked packer={packer_id} mode={mode}")
        assert drv[a[0]] == -1 and (drv[a[1:]] == -2).all()
        (z2, d2, e2, o2, v2), snap2, _, _ = run_groups(packer, case, without, packer_id, mode)
        assert np.array_equal(zone[others], z2) and np.array_equal(drv[others], d2)


@pytest.mark.parametrize("packer_id", PACKERS)
def test_one_instance_group_is_the_single_group_entry(packer, alone, packer_id):
    """n_instance_groups = 1: outputs, availability and gp_stats identical to gp_pack_fifo_zones / gp_pack_fifo_az_aware."""
    rng = np.random.default_rng(9600 + packer_id)
    case = Case(rng, [5])
    apps = make_apps(rng, 1, 300)
    az = packer_id == AZ_AWARE
    for mode in (1, 2):
        got, snap, st, per = run_groups(packer, case, apps, packer_id, mode)
        kw, _ = case.load(alone, az)
        no_group = {k: v for k, v in apps.items() if k != "group"}
        if az:
            order_d, order_e = case.orders[0]
            want = alone.pack_fifo_az_aware(no_group, mode, order_e, order_d, int(kw["n_zones"][0]))
        else:
            want = alone.pack_fifo_zones(no_group, 0 if packer_id == SINGLE_TIGHT else 2, mode)
        (z1, d1, e1, o1, v1), (z2, d2, e2, o2, v2) = got, want
        assert np.array_equal(z1, z2) and np.array_equal(d1, d2) and np.array_equal(o1, o2)
        assert np.array_equal(v1.view(np.uint64), v2.view(np.uint64))
        for j in np.nonzero(d2 >= 0)[0]:                                # ExecutorNodes are defined for placed drivers
            assert np.array_equal(e1[o1[j]:o1[j + 1]], e2[o2[j]:o2[j + 1]])
        for x, y in zip(snap, alone.get_snapshot()):
            assert np.array_equal(x, y)
        counts = lambda s: {k: v for k, v in s.items() if not k.endswith("_ns")}   # the kernel times differ
        assert counts(st) == counts(alone.stats())


def test_refusals(packer, gangpack):
    rng = np.random.default_rng(9700)
    case = Case(rng, [2, 3])
    apps = make_apps(rng, 2, 20)
    Err = gangpack.native.GangpackError

    def refused(match, apps=apps, packer_id=AZ_AWARE, mode=1, load=True, **change):
        kw, _ = case.load(packer, True) if load else (case.layout(True)[1], None)
        before = packer.get_snapshot()
        kw.update(change)
        with pytest.raises(Err) as ei:
            packer.pack_fifo_zones_groups(apps, packer_id, mode, **kw)
        assert ei.value.status == 1 and match in str(ei.value), str(ei.value)
        for x, y in zip(packer.get_snapshot(), before):
            assert np.array_equal(x, y)

    kw, _ = case.load(packer, True)
    packer.pack_fifo_zones_groups(apps, AZ_AWARE, 1, **kw)               # the well-formed call goes through
    _, kw, _ = case.layout(True)
    bad = dict(apps); bad["group"] = np.where(np.arange(20) == 7, 2, apps["group"]).astype(np.int32)
    refused("outside [0, n_instance_groups)", apps=bad)
    bad = dict(apps); bad["group"] = np.where(np.arange(20) == 3, -1, apps["group"]).astype(np.int32)
    refused("outside [0, n_instance_groups)", apps=bad)
    goff = kw["group_off"]
    refused("group_off must run from 0", group_off=np.array([0, goff[1], goff[2] - 1], np.int32))
    refused("group_off must run from 0", group_off=np.array([1, goff[1], goff[2]], np.int32))
    refused("not monotone", group_off=np.array([0, goff[2] + 1, goff[2]], np.int32))
    refused("n_zones[i]", n_zones=np.array([kw["n_zones"][0], goff[2] - goff[1] + 1], np.int32))
    refused("n_zones[i]", n_zones=np.array([-1, kw["n_zones"][1]], np.int32))
    eo = kw["exec_order"].copy(); e0 = int(kw["exec_off"][1])
    refused("exec_order lists a node twice", exec_order=np.where(np.arange(len(eo)) == 1, eo[0], eo).astype(np.int32))
    swapped = np.concatenate([eo[e0:e0 + 1], eo[1:e0], eo[0:1], eo[e0 + 1:]]).astype(np.int32)
    refused("lists a node of another instance group", exec_order=swapped)
    do = kw["drv_order"]
    refused("does not list as a driver candidate", drv_order=np.where(do == do[0], case.exec_only[0], do).astype(np.int32))
    order_e = case.orders[0][1]
    i, j = [k for k, v in enumerate(order_e) if case.zone_of[v] == 0][:2]   # two executors of zone 0 swapped
    e = eo.copy(); e[i], e[j] = e[j], e[i]
    refused("executor order is not exec_order restricted", exec_order=e)
    refused("order lengths", exec_off=np.array([0, e0, len(eo) - 1], np.int32), exec_order=eo[:-1])
    refused("monotone from 0", exec_off=np.array([0, len(eo) + 1, len(eo)], np.int32))
    refused("needs n_zones", n_zones=None)
    refused("packer must be", packer_id=0)
    refused("FIFO modes", mode=0)
    # single-AZ: more than 64 candidate zones in an instance group
    big = Case(np.random.default_rng(9701), [65, 1])
    bkw, _ = big.load(packer, False)
    before = packer.get_snapshot()
    with pytest.raises(Err) as ei:
        packer.pack_fifo_zones_groups(make_apps(rng, 2, 10), SINGLE_TIGHT, 1, **bkw)
    assert ei.value.status == 1 and "more than 64" in str(ei.value)
    for x, y in zip(packer.get_snapshot(), before):
        assert np.array_equal(x, y)
    # no gp_set_schedulable after the snapshot
    snap, kw, _ = case.layout(True)
    packer.set_snapshot(case.cpu, case.mem, case.gpu, *snap)
    with pytest.raises(Err) as ei:
        packer.pack_fifo_zones_groups(apps, AZ_AWARE, 1, **kw)
    assert ei.value.status == 1 and "gp_set_schedulable first" in str(ei.value)
    # a snapshot laid out on the device: no host copy of the layout
    import torch
    t = lambda a, dt: torch.as_tensor(np.asarray(a), dtype=dt, device="cuda")
    keep = [t(case.cpu, torch.int64), t(case.mem, torch.int64), t(case.gpu, torch.int64), t(snap[2], torch.int32), t(snap[0], torch.int32),
            t(snap[3], torch.int32), t(snap[1], torch.int32)]
    packer.set_snapshot_device(*keep)
    packer.set_schedulable(case.sc, case.sm, case.sg)
    for pid in PACKERS:
        with pytest.raises(Err) as ei:
            packer.pack_fifo_zones_groups(apps, pid, 1, **(kw if pid == AZ_AWARE else {"group_off": kw["group_off"]}))
        assert ei.value.status == 1 and "laid out by gp_set_snapshot" in str(ei.value)
    packer.synchronize()
