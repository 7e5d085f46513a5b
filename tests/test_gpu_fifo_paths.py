"""The two device implementations of one fitEarlierDrivers decision (internal/extender/resource.go:224-262) in
gp_pack_fifo_cta, each against the closed-form oracle at the shapes that reach them:

* warp first (default): warp 0 decides an application alone from its per-shape cursors and hands it to the whole CTA
  (general arithmetic class, more than 0xFFFF executors, a first fit or first room more than 1 024 positions past its
  cursor, executors that do not fit with the first fitting driver);
* GANGPACK_FIFO_WARP=0: the whole CTA decides every application (test_cta_path_alone runs this file again that way).

Every case runs tightly-pack and distribute-evenly in both accounting modes and compares every driver_node (incl. -1 / -2),
every ExecutorNodes slice and the final snapshot, per instance group; cases under 400 nodes also go through the literal
restatement.  Each case asserts through stats()["scan_path_apps"] (applications decided by the whole CTA) that it
reaches the path it is named after."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import assert_same_results, fifo_vs_closed, group_slices, literal_fifo

pytestmark = pytest.mark.gpu

WARP_FIRST = os.environ.get("GANGPACK_FIFO_WARP", "1") != "0"
GI, MI = 1 << 30, 1 << 20


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def _apps(q, **cols):
    a = {"drv_cpu": 100, "drv_mem": 128 * MI, "drv_gpu": 0, "exe_cpu": 1000, "exe_mem": GI, "exe_gpu": 0, "count": 1, "young": 1}
    a.update(cols)
    out = {k: np.broadcast_to(np.asarray(v, np.int64), (q,)).copy() for k, v in a.items()}
    out["count"] = out["count"].astype(np.int32)
    out["young"] = out["young"].astype(np.uint8)
    if "group" in out:
        out["group"] = out["group"].astype(np.int32)
    return out


def _case(cpu, mem, gpu, apps, eorder=None, dorder=None, eoff=None, doff=None, check=None):
    n = len(cpu)
    eorder = np.arange(n, dtype=np.int32) if eorder is None else np.asarray(eorder, np.int32)
    dorder = eorder if dorder is None else np.asarray(dorder, np.int32)
    return dict(cpu=np.asarray(cpu, np.int64), mem=np.asarray(mem, np.int64), gpu=np.asarray(gpu, np.int64), apps=apps,
                eorder=eorder, dorder=dorder, eoff=eoff, doff=doff, check=check)


def _mixed(esc, q_eval, dn, apps, algo):
    assert 0 < esc < q_eval, (esc, q_eval)


# ---- cases ------------------------------------------------------------------------------------------------------------
def window_exec(algo):
    """Identical orders, 4 000 nodes: the first 1 500 have room for 1-core executors only, the rest for 16.  The 1-core
    batch minimum keeps the front alive, so a 2-core executor shape scans past the warp's 1 024-node budget, hands off,
    keeps its cursor at the window end, and every later application of that shape resolves on the warp path from there."""
    n = 4000
    cpu = np.where(np.arange(n) < 1500, 1500, 16000)
    i = np.arange(300)
    two = i % 2 == 1
    apps = _apps(300, exe_cpu=np.where(two, 2000, 1000), count=np.where(two, 1 + (i * 5) % 6, 1 + (i * 7) % 3),
                 young=(i % 5 != 0))

    def check(esc, q_eval, dn, apps, algo):
        assert 0 < esc <= 30, esc               # one hand-off per cursor, not one per 2-core application
        assert (dn[two] >= 0).all()
    return _case(cpu, np.full(n, 64 * GI), np.zeros(n), apps, check=check)


def window_drv(algo):
    """A large driver shape whose first fitting candidate is 1 500 entries deep (kWarpWinD hand-off), alternating with a
    small driver shape that fits at the front."""
    n = 3000
    cpu = np.where(np.arange(n) < 1500, 2000, 16000)
    i = np.arange(300)
    apps = _apps(300, drv_cpu=np.where(i % 2 == 1, 8000, 500), drv_mem=256 * MI, count=1 + i % 4)

    def check(esc, q_eval, dn, apps, algo):
        _mixed(esc, q_eval, dn, apps, algo)
        big = apps["drv_cpu"] == 8000
        assert (dn[big] >= 1500).all() and (dn[~big] < 1500).all()
    return _case(cpu, np.full(n, 64 * GI), np.zeros(n), apps, check=check)


def multi_step(algo):
    """Gangs that need 2-30 warp steps of 32 nodes (the commit from the cache of takes) next to gangs that fit in one
    step (the commit from registers).  Nodes hold three executors, so takes above 1 tell the two accounting modes apart."""
    n = 10000
    i = np.arange(120)
    large = i % 4 == 1
    big = 97 + (i * 389) % 1104 if algo == 0 else 33 + (i * 389) % 668
    apps = _apps(120, count=np.where(large, big, 1 + (i * 13) % 40))

    def check(esc, q_eval, dn, apps, algo):
        assert esc <= 12, esc
        assert (dn[large] >= 0).sum() >= 20
    return _case(np.full(n, 3000), np.full(n, 64 * GI), np.zeros(n), apps, check=check)


def cursor_table(D, E, burst):
    """D driver and E executor request tuples (31 / 32 / 33 / 100: the table of 32 cursors not full, full, overflowing).
    Consecutive tuples differ only in the gpu request; tuples 24 apart differ by one byte of memory.  Every 13th
    application is of the general arithmetic class (a 1-millicore executor), so the CTA decides it and the cursors
    must survive that decision."""
    def build(algo):
        rng = np.random.default_rng(900 + D + E + burst)
        n, q = 360, 600
        i = np.arange(q)
        ei = (i // 8) % E if burst else i % E
        di = (i // 5) % D if burst else (i * 7 + i // E) % D
        eb, db = ei // 2, di // 2
        exe_cpu = 250 * (1 + eb % 4)
        apps = _apps(q, exe_cpu=np.where(i % 13 == 6, 1, exe_cpu), exe_mem=(1 << 28) * (1 + (eb // 4) % 3) + eb // 12,
                     exe_gpu=ei % 2, drv_cpu=100 * (1 + db % 5), drv_mem=(1 << 26) * (1 + (db // 5) % 4) + db // 20,
                     drv_gpu=di % 2, count=1 + (i * 11) % 5, young=(i % 17 != 0))
        dorder = None if burst else rng.permutation(n)
        # memory below 2^32 bytes: odd executor memory stays in the fast class
        return _case(np.full(n, 6000), np.full(n, 15 * 256 * MI), rng.integers(0, 9, n), apps, dorder=dorder, check=_mixed)
    return build


def arith_mixed(algo):
    """Memory availabilities above 2^40, odd executor memory above 2^33 (general class: the CTA decides every such
    application) interleaved with fast-class applications whose cursors must stay valid across those hand-offs."""
    rng = np.random.default_rng(31)
    n = 380
    i = np.arange(400)
    gen = i % 3 == 0
    apps = _apps(400, exe_cpu=1000 * (1 + i % 3), exe_mem=np.where(gen, (1 << 33) + 1 + 2 * (i % 5), GI * (1 + i % 4)),
                 drv_cpu=500, drv_mem=GI, count=1 + i % 8)

    def check(esc, q_eval, dn, apps, algo):
        assert ((dn != -2) & gen).sum() <= esc < q_eval, esc
    return _case(np.full(n, 32000), (1 << 40) + rng.integers(0, 1024, n) * GI, np.zeros(n), apps, check=check)


LARGE_COUNTS = [3, 65535, 5, 65536, 2, 70000, 1, 1 << 20, 4, 65535, 7, 100]


def large_gangs(algo):
    """Executors of 2 m / 1 MiB on nodes with 64 000 m free: counts around the uint16 take cache (65 535 / 65 536), above
    it, and at the FIFO limit 2^20.  Counts above 0xFFFF go to the CTA, which then runs without its capacity cache."""
    n = 100
    counts = np.array(LARGE_COUNTS)
    apps = _apps(len(counts), exe_cpu=2, exe_mem=MI, drv_mem=64 * MI, count=counts)

    def check(esc, q_eval, dn, apps, algo):
        assert ((dn != -2) & (counts > 0xFFFF)).sum() <= esc < q_eval, esc
    return _case(np.full(n, 64000), np.full(n, 64 * GI), np.zeros(n), apps, check=check)


def cta_cache_limit(algo):
    """16 000 nodes, every 20th can host executors: the big gangs span more than kFifoCache (12 288) positions, so the
    optimistic pass gives up and phases 1-3 run past the cached prefix; slots beyond 11 776 come from global memory."""
    n = 16000
    host = np.arange(n) % 20 == 0
    i = np.arange(40)
    big = np.isin(i, [3, 17, 30])
    apps = _apps(40, count=np.where(big, 45000 if algo == 0 else 700, 1 + i % 9))

    def check(esc, q_eval, dn, apps, algo):
        assert ((dn != -2) & big).sum() <= esc < q_eval, esc
        assert dn[3] >= 0
    return _case(np.where(host, 64000, 500), np.where(host, 128 * GI, 4 * GI), np.zeros(n), apps, check=check)


def evenly_rounds(algo):
    """A tight cluster of 60 nodes and gangs of 60-150: fewer hosting nodes than executors (m1 <= k), so
    distribute-evenly needs several rounds (the list path of fifo_app)."""
    rng = np.random.default_rng(5)
    n = 60
    i = np.arange(100)
    apps = _apps(100, count=np.where(i % 3 == 0, 60 + (i * 37) % 91, 1 + i % 3))
    return _case(1000 * rng.integers(4, 13, n), np.full(n, 32 * GI), np.zeros(n), apps, check=_mixed)


def three_phase(algo):
    """8 groups of 30 executor nodes (room for two executors each) and 10 driver-only nodes behind them in the driver
    order.  A gang of 60 does not fit with its driver on the first candidate; only a driver-only node works (phase 2)."""
    G, ne, nd = 8, 30, 40
    cpu = np.tile(np.r_[np.full(ne, 2000), np.full(nd - ne, 1000)], G)
    eorder = np.concatenate([g * nd + np.arange(ne) for g in range(G)])
    dorder = np.arange(G * nd)
    pattern = np.array([60, 0, 10, 45, 3, 0])
    q = G * len(pattern)
    i = np.arange(q)
    apps = _apps(q, drv_cpu=1000, count=pattern[i // G], group=i % G)

    def check(esc, q_eval, dn, apps, algo):
        assert G <= esc < q_eval, esc
        assert (dn[:G] % nd >= ne).all()             # the first gang of every group: its driver on a driver-only node
    return _case(cpu, np.full(G * nd, 16 * GI), np.zeros(G * nd), apps, eorder=eorder, dorder=dorder,
                 eoff=np.arange(G + 1) * ne, doff=np.arange(G + 1) * nd, check=check)


def staging(ne, variant):
    """Groups at the shared-memory staging boundary (11 776 slots): identical orders with 11 775 / 11 776 / 11 777
    executor slots, driver-only slots (nd > ne), a permuted driver order.  Only the last 300 executor slots can host
    executors, so every gang lands on both sides of the boundary."""
    def build(algo):
        extra = 40 if variant == "drv_only" else 0
        n = ne + extra
        cpu = np.where(np.arange(n) < ne - 300, 500, 3000)
        cpu[ne:] = 1000
        i = np.arange(200)
        apps = _apps(200, count=1 + (i * 5) % 8, young=(i % 10 != 9))
        eorder = np.arange(ne)
        dorder = np.arange(n) if variant == "drv_only" else (np.random.default_rng(ne).permutation(ne) if variant == "perm" else None)

        def check(esc, q_eval, dn, apps, algo):
            _mixed(esc, q_eval, dn, apps, algo)
        return _case(cpu, np.full(n, 64 * GI), np.zeros(n), apps, eorder=eorder, dorder=dorder, check=check)
    return build


def dead_prefix(algo):
    """Hungry gangs (one 4-core executor per node) fill the front of the order completely, then small gangs follow with
    young applications that fit nowhere interleaved; more hungry gangs later.  The dead prefix moves in the middle of the
    queue."""
    n = 3000
    i = np.arange(400)
    hungry = (i < 40) | (i % 50 == 25)
    nofit_exe = i % 7 == 3
    nofit_drv = i % 11 == 5
    apps = _apps(400, exe_cpu=np.where(hungry, 4000, 1000), count=np.where(hungry, 30, np.where(nofit_exe, 60000, 1 + i % 5)),
                 drv_cpu=np.where(nofit_drv & ~hungry, 8000, 100), young=np.where(hungry, 0, 1))

    def check(esc, q_eval, dn, apps, algo):
        _mixed(esc, q_eval, dn, apps, algo)
        assert (dn[nofit_exe & ~hungry] == -1).all() and (dn[:40] >= 0).all()
    return _case(np.full(n, 4000), np.full(n, 64 * GI), np.zeros(n), apps, check=check)


def gpu_dim(negative, perm):
    """gpu requests on a cluster with gpus; with `negative`, some gpu availabilities are below zero in the snapshot
    (every application then reads the gpu dimension).  Both views: identical orders and a permuted driver order."""
    def build(algo):
        rng = np.random.default_rng(70 + negative + 2 * perm)
        n, q = 300, 300
        gpu = rng.integers(0, 5, n)
        if negative:
            gpu = np.where(rng.random(n) < 0.1, -1, gpu)
        i = np.arange(q)
        apps = _apps(q, exe_cpu=np.where(i % 10 == 4, 1, 250 * (1 + i % 4)), exe_mem=(1 << 28) * (1 + i % 5), exe_gpu=i % 3 == 0,
                     drv_cpu=500, drv_mem=1 << 29, drv_gpu=i % 5 == 0, count=1 + i % 6, young=(i % 13 != 0))
        eorder = rng.permutation(n)
        dorder = rng.permutation(n) if perm else eorder
        return _case(500 * rng.integers(2, 17, n), (1 << 29) * rng.integers(4, 33, n), gpu, apps, eorder=eorder, dorder=dorder,
                     check=_mixed)
    return build


def many_groups(algo):
    """200 groups of 20-300 nodes (more CTAs than SMs), the queue interleaving 170 of them, 30 groups without
    applications; random shapes (a quarter of them in the general class)."""
    from helpers import random_apps
    rng = np.random.default_rng(200)
    G = 200
    sizes = rng.integers(20, 301, G)
    n = int(sizes.sum())
    eoff = np.r_[0, np.cumsum(sizes)].astype(np.int32)
    cpu = 1000 * rng.integers(1, 17, n)
    mem = GI * rng.integers(2, 65, n)
    eorder, dorder, doff = [], [], [0]
    for g in range(G):
        members = np.arange(eoff[g], eoff[g + 1])
        eorder.append(members[np.lexsort((members, cpu[members], mem[members]))])
        d = rng.permutation(members)[: max(1, int(0.7 * len(members)))]
        dorder.append(d)
        doff.append(doff[-1] + len(d))
    q = 4000
    apps = random_apps(rng, q)
    apps["group"] = rng.choice(rng.permutation(G)[:170], q).astype(np.int32)
    apps["young"] = (rng.random(q) < 0.7).astype(np.uint8)
    return _case(cpu, mem, np.zeros(n), apps, eorder=np.concatenate(eorder), dorder=np.concatenate(dorder),
                 eoff=eoff, doff=np.asarray(doff, np.int32), check=_mixed)


CASES = {
    "window_exec": window_exec,
    "window_drv": window_drv,
    "multi_step": multi_step,
    "cursors_31x33": cursor_table(31, 33, False),
    "cursors_32x32_burst": cursor_table(32, 32, True),
    "cursors_33x31_burst": cursor_table(33, 31, True),
    "cursors_100x100": cursor_table(100, 100, False),
    "arith_mixed": arith_mixed,
    "large_gangs": large_gangs,
    "cta_cache_limit": cta_cache_limit,
    "evenly_rounds": evenly_rounds,
    "three_phase": three_phase,
    "staging_11775": staging(11775, "ident"),
    "staging_11776": staging(11776, "ident"),
    "staging_11777": staging(11777, "ident"),
    "staging_drv_only": staging(11776, "drv_only"),
    "staging_perm": staging(11776, "perm"),
    "dead_prefix": dead_prefix,
    "gpu_dim": gpu_dim(False, False),
    "gpu_negative_perm": gpu_dim(True, True),
    "many_groups": many_groups,
}


@pytest.mark.parametrize("name", list(CASES))
def test_fifo_path(oracle, packer, name):
    for algo in (0, 1):
        c = CASES[name](algo)
        a = c["apps"]
        single = c["eoff"] is None
        eoff = np.array([0, len(c["eorder"])], np.int32) if single else c["eoff"]
        doff = np.array([0, len(c["dorder"])], np.int32) if single else c["doff"]
        for mode in (1, 2):
            label = f"{name} algo {algo} mode {mode} warp_first {WARP_FIRST}"
            if single:
                packer.set_snapshot(c["cpu"], c["mem"], c["gpu"], c["eorder"], c["dorder"])
            else:
                packer.set_snapshot(c["cpu"], c["mem"], c["gpu"], c["eorder"], c["dorder"], eoff, doff)
            got = packer.pack_batch(a, algo, mode)
            esc = int(packer.stats()["scan_path_apps"])
            fc, fm, fg = packer.get_snapshot()
            final = fifo_vs_closed(oracle, algo, mode, c["cpu"], c["mem"], c["gpu"], c["eorder"], c["dorder"], eoff, doff, a, got, label)
            assert np.array_equal(fc, final[0]) and np.array_equal(fm, final[1]) and np.array_equal(fg, final[2]), label
            dn = got[0]
            q_eval = int((dn != -2).sum())
            assert (dn >= 0).any(), label
            if WARP_FIRST:
                c["check"](esc, q_eval, dn, a, algo)
            else:
                assert esc == q_eval, (label, esc, q_eval)
            if len(c["cpu"]) <= 400:
                group = a.get("group", np.zeros(len(dn), np.int32))
                avail = (c["cpu"], c["mem"], c["gpu"])
                for g in range(len(eoff) - 1):
                    sel = np.nonzero(group == g)[0]
                    sub = {k: np.asarray(v)[sel] for k, v in a.items()}
                    want, avail = literal_fifo(oracle, algo, mode, avail[0], avail[1], avail[2], c["dorder"][doff[g]:doff[g + 1]],
                                               c["eorder"][eoff[g]:eoff[g + 1]], sub, sub["young"])
                    assert_same_results(group_slices(*got, sel), want, f"{label} literal group {g}")
                assert all(np.array_equal(x, y) for x, y in zip(avail, final)), label


def test_counts_above_fifo_limit_refused(packer, gangpack):
    """2^20 executors is the FIFO limit (block-wide uint32 sums of clamped capacities); one more is refused."""
    n = 100
    packer.set_snapshot(np.full(n, 64000), np.full(n, 64 * GI), np.zeros(n), np.arange(n, dtype=np.int32), np.arange(n, dtype=np.int32))
    for mode in (1, 2):
        with pytest.raises(gangpack.native.GangpackError) as e:
            packer.pack_batch(_apps(3, exe_cpu=2, exe_mem=MI, count=[4, (1 << 20) + 1, 4]), 0, mode)
        assert e.value.status == 6
    dn, _, _ = packer.pack_batch(_apps(2, exe_cpu=2, exe_mem=MI, count=[1 << 20, 4]), 0, 1)
    assert (dn >= 0).all()


def test_cta_path_alone():
    """The same cases with GANGPACK_FIFO_WARP=0: the whole CTA decides every application."""
    if not WARP_FIRST:
        pytest.skip("already running with GANGPACK_FIFO_WARP=0")
    env = dict(os.environ, GANGPACK_FIFO_WARP="0")
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-q", "-x",
                        "-k", "not test_cta_path_alone"], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]
