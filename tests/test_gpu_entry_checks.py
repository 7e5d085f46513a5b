"""The host checks of the reservation-driven C ABI entries, called through ctypes with the binding's structs so that arrays can
be NULL: each malformed input is refused with its status and a message that names the entry called, and a valid call right
after it succeeds.  A refused gp_prepare_cluster_zones leaves the context as it was, held az-aware orders included."""
import ctypes as C

import numpy as np
import pytest

import k8s_spark_scheduler_b200 as g

pytestmark = pytest.mark.gpu

native = g.native
I64, I32, U8 = np.int64, np.int32, np.uint8
N = 4                                   # nodes of every valid input
_keep = []                              # arrays the structs of the current call point at


def _a(v, dt):
    a = np.ascontiguousarray(v, dtype=dt)
    _keep.append(a)
    return a.ctypes.data


def _opt(v, dt):
    return None if v is None else _a(v, dt)


def _out(n, dt=I64):
    return _a(np.zeros(n), dt)


def ref(s):
    return None if s is None else C.byref(s)


def usage(**kw):
    u = native.gp_usage_input(n_nodes=N, alloc_cpu_milli=_a([8000] * N, I64), alloc_mem_bytes=_a([16 << 30] * N, I64),
                              alloc_gpu=_a([1, 0, 2, 0], I64), n_reservations=3, res_node=_a([0, 2, -1], I32),
                              res_cpu_milli=_a([1000, 500, 100], I64), res_mem_bytes=_a([1 << 30, 1 << 29, 1 << 20], I64))
    for k, v in kw.items():
        setattr(u, k, v)
    return u


def sort(avail=False, zone_id=(0, 1, 0, 1), name_rank=(3, 1, 0, 2)):
    s = native.gp_sort_input(n_nodes=N, n_zones=2, zone_id=_a(zone_id, I32), name_rank=_a(name_rank, I32))
    if avail:
        s.avail_cpu_milli, s.avail_mem_bytes = _a([4000, 3000, 2000, 1000], I64), _a([8 << 30] * N, I64)
    return s


def resched(cpu=(100, 200), mem=(1 << 20, 1 << 21), gpu=None, min_frag=0, host_off=None, host_nodes=None):
    return native.gp_reschedule(n_execs=len(cpu), exe_cpu_milli=_a(cpu, I64), exe_mem_bytes=_a(mem, I64), exe_gpu=_opt(gpu, I64),
                                min_frag=min_frag, host_off=_opt(host_off, I64), host_nodes=_opt(host_nodes, I32))


def reconcile(L, h, u, r):
    """gp_reconcile_find_nodes with r's request columns, one executor per application, one instance group"""
    q = r.n_execs
    nodes = native.gp_reconcile_nodes(n_groups=1, node_group=_a([0] * N, I32), creation=_a(np.arange(N), I64))
    a = native.gp_apps(n_apps=q, exe_cpu_milli=r.exe_cpu_milli, exe_mem_bytes=r.exe_mem_bytes, exe_gpu=r.exe_gpu,
                       exe_count=_a([1] * q, I32))
    out = native.gp_reconcile_results(placed=_out(q, I32), executor_nodes=_out(q, I32), executor_nodes_cap=q)
    return L.gp_reconcile_find_nodes(h, ref(u), C.byref(nodes), C.byref(a), C.byref(out))


RUN = {
    "gp_build_availability": lambda L, h, u, s, r: L.gp_build_availability(h, ref(u), *[_out(N) for _ in range(6)]),
    "gp_build_reschedule_availability": lambda L, h, u, s, r: L.gp_build_reschedule_availability(h, ref(u), *[_out(N) for _ in range(3)]),
    "gp_prepare_cluster": lambda L, h, u, s, r: L.gp_prepare_cluster(h, ref(u), ref(s), C.byref(C.c_int32()), C.byref(C.c_int32())),
    "gp_prepare_cluster_zones": lambda L, h, u, s, r: L.gp_prepare_cluster_zones(
        h, ref(u), ref(s), C.byref(native.gp_zone_layout(kind=native.LAYOUT_AZ_AWARE))),
    "gp_reschedule_from_reservations": lambda L, h, u, s, r: L.gp_reschedule_from_reservations(
        h, ref(u), ref(s), None, ref(r), _out(r.n_execs, I32), _out(r.n_execs, U8)),
    "gp_reconcile_find_nodes": lambda L, h, u, s, r: reconcile(L, h, u, r),
    "gp_reschedule_executors": lambda L, h, u, s, r: L.gp_reschedule_executors(h, ref(r), _out(r.n_execs, I32)),
    "gp_potential_nodes": lambda L, h, u, s, r: L.gp_potential_nodes(h, ref(s), _out(N, I32), C.byref(C.c_int32()), _out(N, I32),
                                                                    C.byref(C.c_int32())),
}
USAGE_ENTRIES = ["gp_build_availability", "gp_build_reschedule_availability", "gp_prepare_cluster", "gp_prepare_cluster_zones",
                 "gp_reschedule_from_reservations", "gp_reconcile_find_nodes"]
SORT_ENTRIES = ["gp_potential_nodes", "gp_prepare_cluster", "gp_prepare_cluster_zones", "gp_reschedule_from_reservations"]
REQUEST_ENTRIES = ["gp_reschedule_executors", "gp_reschedule_from_reservations", "gp_reconcile_find_nodes"]
CSR_ENTRIES = ["gp_reschedule_executors", "gp_reschedule_from_reservations"]


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    assert call(p, "gp_prepare_cluster") == 0          # gp_reschedule_executors wants a snapshot (4 nodes, one group)
    yield p
    p.close()


def call(p, entry, u=None, s=None, r=None):
    """one call of `entry`; u / s / r default to valid inputs"""
    try:
        return RUN[entry](native.load(), p._h, usage() if u is None else u,
                          s or sort(avail=entry == "gp_potential_nodes"), r or resched())
    finally:
        _keep.clear()


def refused(p, entry, status, text, **kw):
    assert call(p, entry, **kw) == status
    msg = (native.load().gp_last_error(p._h) or b"").decode()
    assert msg.startswith(entry + ": ") and text in msg, msg
    assert call(p, entry) == 0, (native.load().gp_last_error(p._h) or b"").decode()


USAGE_CASES = {
    "null": lambda: None,
    "negative n_nodes": lambda: usage(n_nodes=-1),
    "negative n_reservations": lambda: usage(n_reservations=-1),
    "no alloc_cpu_milli": lambda: usage(alloc_cpu_milli=None),
    "no alloc_mem_bytes": lambda: usage(alloc_mem_bytes=None),
    "no res_node": lambda: usage(res_node=None),
    "no res_cpu_milli": lambda: usage(res_cpu_milli=None),
    "no res_mem_bytes": lambda: usage(res_mem_bytes=None),
}


@pytest.mark.parametrize("case", list(USAGE_CASES))
@pytest.mark.parametrize("entry", USAGE_ENTRIES)
def test_usage_shape(packer, entry, case):
    u = USAGE_CASES[case]()
    if u is None:                       # an explicit NULL: call() would substitute the valid default
        assert RUN[entry](native.load(), packer._h, None, sort(), resched()) == 1
        _keep.clear()
        msg = native.load().gp_last_error(packer._h).decode()
        assert msg.startswith(entry + ": ") and "missing arrays" in msg, msg
        assert call(packer, entry) == 0
    else:
        refused(packer, entry, 1, "missing arrays", u=u)


SORT_CASES = {
    "zone_id >= n_zones": (dict(zone_id=(0, 2, 1, 0)), "zone_id out of range"),
    "negative zone_id": (dict(zone_id=(0, -1, 1, 0)), "zone_id out of range"),
    "name_rank >= n_nodes": (dict(name_rank=(0, 4, 1, 2)), "name_rank out of range"),
    "negative name_rank": (dict(name_rank=(0, -1, 1, 2)), "name_rank out of range"),
    "name_rank given twice": (dict(name_rank=(0, 1, 1, 2)), "name_rank is not a permutation"),
    "name_rank all equal": (dict(name_rank=(3, 3, 3, 3)), "name_rank is not a permutation"),
}


@pytest.mark.parametrize("case", list(SORT_CASES))
@pytest.mark.parametrize("entry", SORT_ENTRIES)
def test_sort_ids(packer, entry, case):
    kw, text = SORT_CASES[case]
    refused(packer, entry, 1, text, s=sort(avail=entry == "gp_potential_nodes", **kw))


REQUEST_CASES = {
    "negative cpu": (dict(cpu=(-1, 200)), 1, "negative resource request"),
    "mem >= 2^61": (dict(mem=(1 << 61, 1)), 6, "quantity >= 2^61"),
    "negative gpu": (dict(gpu=(0, -1)), 1, "negative resource request"),
}


@pytest.mark.parametrize("case", list(REQUEST_CASES))
@pytest.mark.parametrize("entry", REQUEST_ENTRIES)
def test_request_domain(packer, entry, case):
    kw, status, text = REQUEST_CASES[case]
    assert call(packer, "gp_prepare_cluster") == 0      # the snapshot gp_reschedule_executors runs against
    refused(packer, entry, status, text, r=resched(**kw))


CSR_CASES = {
    "host_off[0] != 0": (dict(host_off=(1, 1, 2), host_nodes=(0, 1)), "host_off must start at 0"),
    "host_off not monotone": (dict(host_off=(0, 2, 1), host_nodes=(0, 1)), "host_off not monotone"),
    "no host_nodes": (dict(host_off=(0, 1, 2)), "host_nodes missing"),
    "host_nodes >= n_nodes": (dict(host_off=(0, 1, 2), host_nodes=(0, N)), "host_nodes index out of range"),
}


@pytest.mark.parametrize("case", list(CSR_CASES))
@pytest.mark.parametrize("entry", CSR_ENTRIES)
def test_hosting_csr(packer, entry, case):
    kw, text = CSR_CASES[case]
    assert call(packer, "gp_prepare_cluster") == 0      # N nodes bound host_nodes of gp_reschedule_executors
    refused(packer, entry, 1, text, r=resched(min_frag=1, **kw))
    assert call(packer, entry, r=resched(min_frag=1, host_off=(0, 1, 2), host_nodes=(0, 1))) == 0


def test_refused_prepare_keeps_held_orders(packer):
    rng = np.random.default_rng(7)
    n = 64
    alloc = (rng.integers(2, 17, n) * 1000, rng.integers(4, 65, n) << 30, rng.integers(0, 2, n))
    res_node = rng.integers(-1, n, 40).astype(np.int32)
    res = (rng.integers(0, 5, 40) * 500, rng.integers(0, 5, 40) << 29, np.zeros(40, np.int64))
    zid = rng.integers(0, 3, n).astype(np.int32)
    apps = dict(drv_cpu=[1000, 2000, 500, 4000], drv_mem=[1 << 30, 2 << 30, 1 << 29, 8 << 30], exe_cpu=[2000, 1000, 3000, 500],
                exe_mem=[4 << 30, 1 << 30, 2 << 30, 1 << 29], count=[3, 1, 5, 2])
    packer.prepare_cluster_zones(alloc, None, res_node, res, zid, 3, kind=native.LAYOUT_AZ_AWARE)
    want = packer.pack_batch_az_aware(apps)
    with pytest.raises(native.GangpackError) as ei:
        packer.prepare_cluster_zones(alloc, None, res_node, res, np.where(zid == 2, 3, zid).astype(np.int32), 3,
                                     kind=native.LAYOUT_AZ_AWARE)
    assert ei.value.status == 1
    got = packer.pack_batch_az_aware(apps)
    for w, x in zip(want, got):
        assert np.array_equal(np.asarray(w).view(np.uint8), np.asarray(x).view(np.uint8))
