"""How GangPacker marshals the reservation-driven entries and the zone packs into the C ABI, without a GPU.

native._lib is replaced by a fake whose gp_* functions record the entry called and read every argument struct while the
call runs: the n_* fields, which pointers are NULL and the values the others reach."""
import ctypes as C

import numpy as np
import pytest

import k8s_spark_scheduler_b200 as g

native = g.native
I64, I32, U8 = C.c_int64, C.c_int32, C.c_uint8


def _arr(addr, ctype, n):
    return None if not addr else np.ctypeslib.as_array((ctype * n).from_address(addr)).copy()


def _read(s, n, cols):
    """the struct's scalar fields, and each pointer field in `cols` ({name: ctype}) as None (NULL) or its n values"""
    out = {name: getattr(s, name) for name, t in s._fields_ if t is not C.c_void_p}
    out.update({name: _arr(getattr(s, name), t, n) for name, t in cols.items()})
    return out


def usage(u):
    d = _read(u, u.n_nodes, {k: I64 for k in ("alloc_cpu_milli", "alloc_mem_bytes", "alloc_gpu", "overhead_cpu_milli",
                                              "overhead_mem_bytes", "overhead_gpu")})
    d.update(_read(u, u.n_reservations, {"res_node": I32, "res_cpu_milli": I64, "res_mem_bytes": I64, "res_gpu": I64}))
    return d


def sort(s):
    d = _read(s, s.n_nodes, {"avail_cpu_milli": I64, "avail_mem_bytes": I64, "avail_gpu": I64, "zone_id": I32, "name_rank": I32,
                             "is_driver_candidate": U8, "unschedulable": U8, "ready": U8, "driver_label_rank": I32,
                             "executor_label_rank": I32})
    d["undefined_ties"] = bool(s.undefined_ties)
    return d


def apps(a):
    q = a.n_apps
    d = _read(a, q, {k: I64 for k in ("drv_cpu_milli", "drv_mem_bytes", "drv_gpu", "exe_cpu_milli", "exe_mem_bytes", "exe_gpu")})
    d.update(_read(a, q, {"exe_count": I32, "group": I32, "skip_if_no_fit": U8}))
    d["exec_out_off"] = _arr(a.exec_out_off, I64, q + 1)
    return d


def resched(r, n_nodes):
    q = r.n_execs
    d = _read(r, q, {"exe_cpu_milli": I64, "exe_mem_bytes": I64, "exe_gpu": I64, "group": I32})
    d.update(_read(r, n_nodes, {"reserved_cpu_milli": I64, "reserved_mem_bytes": I64, "reserved_gpu": I64}))
    d["host_off"] = _arr(r.host_off, I64, q + 1)
    d["host_nodes"] = _arr(r.host_nodes, I32, int(d["host_off"][-1]) or 1) if r.host_off else bool(r.host_nodes)
    return d


def zone_results(r):
    return dict(cap=r.executor_nodes_cap, null=[not getattr(r, k) for k in ("zone", "driver_node", "executor_nodes", "avg_efficiency")])


def byref_obj(arg):
    return None if arg is None else arg._obj


class FakeLib:
    """Stands in for libgangpack.so: each gp_* call is read by READERS[name] while it runs and returns GP_OK."""

    def __init__(self):
        self.calls = []
        self.n_nodes = 0

    def __getattr__(self, name):
        if not name.startswith("gp_"):
            raise AttributeError(name)

        def call(*args):
            reader = READERS.get(name)
            self.calls.append((name, reader(self, *args[1:]) if reader else None))
            return 0
        return call

    def only(self, name):
        got = [c for c in self.calls if c[0] not in ("gp_create", "gp_destroy")]
        assert [c[0] for c in got] == [name]
        self.calls.clear()
        return got[0][1]


READERS = {
    "gp_build_availability": lambda f, ui, *outs: dict(usage=usage(byref_obj(ui)), outs=[bool(o) for o in outs]),
    "gp_build_reschedule_availability": lambda f, ui, *outs: dict(usage=usage(byref_obj(ui)), outs=[bool(o) for o in outs]),
    "gp_reschedule_executors": lambda f, r, out: dict(r=resched(byref_obj(r), f.n_nodes), out=bool(out)),
    "gp_reschedule_from_reservations": lambda f, ui, si, scope, r, out, amb: dict(
        usage=usage(byref_obj(ui)), sort=sort(byref_obj(si)), r=resched(byref_obj(r), 0), out=bool(out), amb=bool(amb),
        scope=None if scope is None else dict(keep=byref_obj(scope).keep_topology_zone,
                                              tz=_arr(byref_obj(scope).topology_zone, I32, byref_obj(ui).n_nodes))),
    "gp_prepare_cluster": lambda f, ui, si, nd, ne: dict(usage=usage(byref_obj(ui)), sort=sort(byref_obj(si)), counts=[nd is not None, ne is not None]),
    "gp_prepare_cluster_zones": lambda f, ui, si, lo: dict(
        usage=usage(byref_obj(ui)), sort=sort(byref_obj(si)), kind=byref_obj(lo).kind,
        null=[not getattr(byref_obj(lo), k) for k in ("zone_of_group", "exec_off", "exec_order", "drv_off", "drv_order")]),
    "gp_potential_nodes": lambda f, si, d, nd, e, ne: dict(sort=sort(byref_obj(si)), outs=[bool(d), bool(e)]),
    "gp_pack_batch_zones": lambda f, a, algo, r: dict(apps=apps(byref_obj(a)), args=[algo], r=zone_results(byref_obj(r))),
    "gp_pack_fifo_zones": lambda f, a, algo, mode, r: dict(apps=apps(byref_obj(a)), args=[algo, mode], r=zone_results(byref_obj(r))),
    "gp_pack_fifo_az_aware": lambda f, a, mode, o, r: dict(apps=apps(byref_obj(a)), args=[mode], orders=orders(byref_obj(o)),
                                                           r=zone_results(byref_obj(r))),
    "gp_pack_batch_az_aware": lambda f, a, o, r: dict(apps=apps(byref_obj(a)), args=[], orders=orders(byref_obj(o)),
                                                      r=zone_results(byref_obj(r))),
    "gp_reserve_placements": lambda f, a, r, sub, t: dict(apps=apps(byref_obj(a)), sub=sub, cap=byref_obj(r).executor_nodes_cap,
                                                          rows_cap=byref_obj(t).rows_cap),
    "gp_packing_efficiency": lambda f, a, algo, r, charged, avg: dict(apps=apps(byref_obj(a)), args=[algo, charged],
                                                                      cap=byref_obj(r).executor_nodes_cap, avg=bool(avg)),
    "gp_exceeds_cluster_capacity": lambda f, nd, a, packer, out: dict(apps=apps(byref_obj(a)), n_nodes=byref_obj(nd).n_nodes,
                                                                      packer=packer, out=bool(out)),
    "gp_reconcile_find_nodes": lambda f, ui, nd, a, r: dict(
        usage=usage(byref_obj(ui)), apps=apps(byref_obj(a)), n_groups=byref_obj(nd).n_groups,
        node_group=_arr(byref_obj(nd).node_group, I32, byref_obj(ui).n_nodes), cap=byref_obj(r).executor_nodes_cap,
        avail_null=[not getattr(byref_obj(r), k) for k in ("avail_cpu_milli", "avail_mem_bytes", "avail_gpu")]),
}


def orders(o):
    if o is None:
        return None
    return dict(n_zones=o.n_zones, exec_order=_arr(o.exec_order, I32, o.n_exec), drv_order=_arr(o.drv_order, I32, o.n_drv))


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(native, "_lib", f)
    return f


@pytest.fixture
def packer(fake):
    return native.GangPacker()


ALLOC = ([8000, 4000, 2000], [1 << 33, 1 << 32, 1 << 31], [1, 0, 2])
OVER = ([100, 0, 50], [1 << 20, 0, 0], [0, 0, 0])
RNODE = [2, 0, -1, 2]
RES = ([500, 250, 100, 1000], [1 << 28, 1 << 27, 1 << 26, 1 << 29], [0, 1, 0, 0])


def eq(a, b):
    return a is None and b is None or (a is not None and b is not None and np.array_equal(a, np.asarray(b)))


def check_usage(u, alloc=ALLOC, over=OVER, rnode=RNODE, res=RES):
    assert (u["n_nodes"], u["n_reservations"]) == (len(alloc[0]), len(rnode))
    names = ("cpu_milli", "mem_bytes", "gpu")
    for i, k in enumerate(names):
        assert eq(u["alloc_" + k], alloc[i] if i < len(alloc) else None), k
        assert eq(u["overhead_" + k], over[i] if over is not None and i < len(over) else None), k
        assert eq(u["res_" + k], res[i] if i < len(res) else None), k
    assert eq(u["res_node"], rnode)


ZID, RANK, CAND, UNS, READY, LRD, LRE = [1, 0, 1], [2, 0, 1], [1, 0, 1], [0, 0, 1], [1, 1, 0], [0, -1, 1], [1, 1, -1]


def check_sort(s, n=3, n_zones=2, cand=True, lrd=True, avail=None, ties=True):
    assert (s["n_nodes"], s["n_zones"]) == (n, n_zones)
    assert eq(s["zone_id"], ZID) and eq(s["name_rank"], RANK) and eq(s["unschedulable"], UNS) and eq(s["ready"], READY)
    assert eq(s["executor_label_rank"], LRE)
    assert eq(s["is_driver_candidate"], CAND if cand else None)
    assert eq(s["driver_label_rank"], LRD if lrd else None)
    for i, k in enumerate(("avail_cpu_milli", "avail_mem_bytes", "avail_gpu")):
        assert eq(s[k], avail[i] if avail is not None else None), k
    assert s["undefined_ties"] == ties


def test_build_availability(packer, fake):
    packer.build_availability(ALLOC, OVER, RNODE, RES)
    got = fake.only("gp_build_availability")
    check_usage(got["usage"])
    assert got["outs"] == [True] * 6
    packer.build_availability(ALLOC, None, RNODE, RES)
    check_usage(fake.only("gp_build_availability")["usage"], over=None)


def test_build_reschedule_availability(packer, fake):
    packer.build_reschedule_availability(ALLOC, OVER, RNODE, RES)
    got = fake.only("gp_build_reschedule_availability")
    check_usage(got["usage"])
    assert got["outs"] == [True] * 3


def test_reschedule_executors(packer, fake):
    fake.n_nodes = 3
    exe = ([100, 200], [1 << 20, 1 << 21], [0, 1])
    packer.reschedule_executors(exe, min_frag=True, group=[0, 1], reserved=([1, 2, 3], [4, 5, 6], [0, 0, 1]), hosting=[[2], [0, 1]])
    r = fake.only("gp_reschedule_executors")
    assert r["out"]
    r = r["r"]
    assert (r["n_execs"], r["min_frag"]) == (2, 1)
    assert eq(r["exe_cpu_milli"], exe[0]) and eq(r["exe_mem_bytes"], exe[1]) and eq(r["exe_gpu"], exe[2]) and eq(r["group"], [0, 1])
    assert eq(r["reserved_cpu_milli"], [1, 2, 3]) and eq(r["reserved_mem_bytes"], [4, 5, 6]) and eq(r["reserved_gpu"], [0, 0, 1])
    assert eq(r["host_off"], [0, 1, 3]) and eq(r["host_nodes"], [2, 0, 1])
    packer.reschedule_executors(exe[:2])
    r = fake.only("gp_reschedule_executors")["r"]
    assert r["min_frag"] == 0 and r["exe_gpu"] is None and r["group"] is None and r["reserved_cpu_milli"] is None
    assert r["host_off"] is None and r["host_nodes"] is False


def test_reschedule_from_reservations(packer, fake):
    exe = ([100, 200], [1 << 20, 1 << 21], None)
    packer.reschedule_from_reservations(ALLOC, OVER, RNODE, RES, exe, min_frag=True, hosting=[[], [1, 2]], zone_id=ZID, n_zones=2,
                                        name_rank=RANK, unschedulable=UNS, ready=READY, executor_label_rank=LRE,
                                        keep_topology_zone=1, topology_zone=[1, 1, 0])
    got = fake.only("gp_reschedule_from_reservations")
    check_usage(got["usage"])
    check_sort(got["sort"], cand=False, lrd=False, ties=False)
    assert got["scope"]["keep"] == 1 and eq(got["scope"]["tz"], [1, 1, 0])
    r = got["r"]
    assert (r["n_execs"], r["min_frag"]) == (2, 1) and r["group"] is None and r["exe_gpu"] is None
    assert eq(r["exe_cpu_milli"], exe[0]) and eq(r["exe_mem_bytes"], exe[1])
    assert r["reserved_cpu_milli"] is None and r["reserved_mem_bytes"] is None and r["reserved_gpu"] is None
    assert eq(r["host_off"], [0, 0, 2]) and eq(r["host_nodes"], [1, 2])
    assert got["out"] and got["amb"]
    packer.reschedule_from_reservations((ALLOC[0], ALLOC[1], None), None, RNODE, (RES[0], RES[1], None), exe)
    got = fake.only("gp_reschedule_from_reservations")
    check_usage(got["usage"], alloc=ALLOC[:2], over=None, res=RES[:2])
    assert got["scope"] is None and got["r"]["host_off"] is None and got["sort"]["n_zones"] == 1
    assert all(got["sort"][k] is None for k in ("zone_id", "name_rank", "unschedulable", "ready", "executor_label_rank"))


def test_prepare_cluster(packer, fake):
    packer.prepare_cluster(ALLOC, OVER, RNODE, RES, ZID, 2, RANK, CAND, UNS, READY, LRD, LRE)
    got = fake.only("gp_prepare_cluster")
    check_usage(got["usage"])
    check_sort(got["sort"], ties=False)
    assert got["counts"] == [True, True]


@pytest.mark.parametrize("layout", [True, False])
def test_prepare_cluster_zones(packer, fake, layout):
    out = packer.prepare_cluster_zones(ALLOC, OVER, RNODE, RES, ZID, 2, RANK, CAND, UNS, READY, LRD, LRE,
                                       kind=native.LAYOUT_SINGLE_AZ, layout=layout)
    got = fake.only("gp_prepare_cluster_zones")
    check_usage(got["usage"])
    check_sort(got["sort"])
    assert got["kind"] == native.LAYOUT_SINGLE_AZ
    assert got["null"] == [False] + [not layout] * 4
    assert len(out["zone_of_group"]) == 3


def test_potential_nodes(packer, fake):
    avail = ([1, 2, 3], [4, 5, 6], [0, 1, 0])
    packer.potential_nodes(avail[0], avail[1], ZID, 2, RANK, CAND, UNS, READY, LRD, LRE, avail_gpu=avail[2])
    got = fake.only("gp_potential_nodes")
    check_sort(got["sort"], avail=avail)
    assert got["outs"] == [True, True]


APPS = dict(drv_cpu=[100, 200, 300], drv_mem=[1 << 20, 1 << 21, 1 << 22], drv_gpu=[0, 1, 0], exe_cpu=[10, 20, 30],
            exe_mem=[1 << 10, 1 << 11, 1 << 12], count=[2, 0, 3], young=[1, 0, 1], group=[0, 1, 0])
OFF = [0, 2, 2, 5]


def check_apps(a, apps=APPS, off=OFF, skip=False, group=False):
    assert a["n_apps"] == len(apps["count"])
    for src, dst in (("drv_cpu", "drv_cpu_milli"), ("drv_mem", "drv_mem_bytes"), ("drv_gpu", "drv_gpu"),
                     ("exe_cpu", "exe_cpu_milli"), ("exe_mem", "exe_mem_bytes"), ("exe_gpu", "exe_gpu")):
        assert eq(a[dst], apps.get(src)), dst
    assert eq(a["exe_count"], apps["count"])
    assert eq(a["skip_if_no_fit"], apps["young"] if skip else None)
    assert eq(a["group"], apps["group"] if group else None)
    assert eq(a["exec_out_off"], off)


ZONE_PACKS = [
    ("pack_batch_zones", lambda p: p.pack_batch_zones(APPS, 2), "gp_pack_batch_zones", [2], False, None),
    ("pack_fifo_zones", lambda p: p.pack_fifo_zones(APPS, 0, 2), "gp_pack_fifo_zones", [0, 2], True, None),
    ("pack_fifo_az_aware", lambda p: p.pack_fifo_az_aware(APPS, 1), "gp_pack_fifo_az_aware", [1], True, False),
    ("pack_fifo_az_aware_orders", lambda p: p.pack_fifo_az_aware(APPS, 2, [2, 0], [1], 1), "gp_pack_fifo_az_aware", [2], True, True),
    ("pack_batch_az_aware", lambda p: p.pack_batch_az_aware(APPS), "gp_pack_batch_az_aware", [], False, False),
    ("pack_batch_az_aware_orders", lambda p: p.pack_batch_az_aware(APPS, [2, 0], [1], 1), "gp_pack_batch_az_aware", [], False, True),
]


@pytest.mark.parametrize("case", ZONE_PACKS, ids=[z[0] for z in ZONE_PACKS])
def test_zone_packs(packer, fake, case):
    _, call, entry, args, skip, with_orders = case
    zone, drv, exe, off, avg = call(packer)
    got = fake.only(entry)
    check_apps(got["apps"], skip=skip)
    assert got["args"] == args
    assert got["r"] == dict(cap=5, null=[False] * 4)
    if with_orders is not None:
        assert (got["orders"] is not None) == with_orders
        if with_orders:
            assert got["orders"]["n_zones"] == 1 and eq(got["orders"]["exec_order"], [2, 0]) and eq(got["orders"]["drv_order"], [1])
    assert eq(off, OFF) and (len(zone), len(drv), len(exe), avg.shape) == (3, 3, 5, (3, 4))


def test_zone_packs_empty(packer, fake):
    empty = dict(drv_cpu=[], drv_mem=[], exe_cpu=[], exe_mem=[], count=[])
    zone, drv, exe, off, avg = packer.pack_batch_zones(empty, 0)
    got = fake.only("gp_pack_batch_zones")
    assert got["apps"]["n_apps"] == 0 and eq(got["apps"]["exec_out_off"], [0]) and got["r"]["cap"] == 1
    assert (len(zone), len(exe), avg.shape) == (0, 0, (0, 4))


def test_reserve_placements(packer, fake):
    packer.reserve_placements(APPS, ([0, -1, 2], [1, 2, 0, 1, 2], OFF), subtract=False)
    got = fake.only("gp_reserve_placements")
    check_apps(got["apps"])
    assert (got["sub"], got["cap"], got["rows_cap"]) == (0, 5, 7)


def test_packing_efficiency(packer, fake):
    packer.packing_efficiency(APPS, ([0, -1, 2], [1, 2, 0, 1, 2], OFF), 2, charged=1)
    got = fake.only("gp_packing_efficiency")
    check_apps(got["apps"])
    assert got["args"] == [2, 1] and got["cap"] == 5 and got["avg"]
    packer.packing_efficiency(APPS, ([0, -1, 2], [], OFF), 0)
    assert fake.only("gp_packing_efficiency")["cap"] == 1


def test_exceeds_cluster_capacity(packer, fake):
    packer.exceeds_cluster_capacity(ALLOC, APPS, native.BP_SINGLE_AZ_TIGHTLY_PACK, overhead=OVER, zone_id=ZID, n_zones=2)
    got = fake.only("gp_exceeds_cluster_capacity")
    check_apps(got["apps"], off=None, group=True)
    assert (got["n_nodes"], got["packer"], got["out"]) == (3, native.BP_SINGLE_AZ_TIGHTLY_PACK, True)


def test_reconcile_find_nodes(packer, fake):
    rapps = dict(exe_cpu=[10, 20, 30], exe_mem=[1 << 10, 1 << 11, 1 << 12], count=[2, 0, 3], group=[0, 1, 0])
    packer.reconcile_find_nodes(ALLOC, OVER, RNODE, RES, [0, 1, 0], [5, 6, 7], rapps, 2)
    got = fake.only("gp_reconcile_find_nodes")
    check_usage(got["usage"])
    check_apps(got["apps"], apps=rapps, group=True)
    assert got["n_groups"] == 2 and eq(got["node_group"], [0, 1, 0]) and got["cap"] == 5 and got["avail_null"] == [False] * 3
    packer.reconcile_find_nodes((ALLOC[0], ALLOC[1], None), None, RNODE, (RES[0], RES[1]), [0, 1, 0], [5, 6, 7],
                                dict(rapps, group=None), 2, exec_cap=9, want_avail=False)
    got = fake.only("gp_reconcile_find_nodes")
    check_usage(got["usage"], alloc=ALLOC[:2], over=None, res=RES[:2])
    assert got["apps"]["group"] is None and got["cap"] == 9 and got["avail_null"] == [True] * 3
