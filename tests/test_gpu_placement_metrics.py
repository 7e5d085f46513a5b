"""gp_placement_metrics[_device]: the Predicate's collocation, executor node count and cross-zone metrics on the device.

Every record is checked against the literal, string-keyed restatement of the three reporters (placement_metrics_ref.literal,
Go map order randomised) for: gp_pack_batch results of the three plain packers, independent and both FIFO modes, on the
synth workloads up to 10 000 nodes x 100 000 applications; single-AZ and az-aware zone results, fallback winners included;
a multi-group FIFO drain after gp_prepare_cluster_groups with instance_group; adversarial rows (rows above the warp path,
every node its own zone, a node table whose bitmap does not fit in shared memory).  The device form on
gp_pack_batch_device outputs equals the host form bit for bit; the call leaves the snapshot and gp_last_stats untouched;
every refusal is covered."""
import numpy as np
import pytest

import placement_metrics_ref as ref

pytestmark = pytest.mark.gpu

INDEPENDENT, FIFO_REFERENCE, FIFO_EXACT = 0, 1, 2
TIGHTLY, EVENLY, MINFRAG = 0, 1, 2
G = 1 << 30
APP_COLS = ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group")


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def labels_of(rng, n, n_labels=4):
    """failure-domain labels: some nodes unlabelled, some literally labelled unknown-zone"""
    out = []
    for r, z in zip(rng.random(n), rng.integers(0, n_labels, n)):
        out.append({} if r < 0.05 else {ref.LABEL_ZONE_FAILURE_DOMAIN: "unknown-zone"} if r < 0.08 else
                   {ref.LABEL_ZONE_FAILURE_DOMAIN: "zone-%d" % z})
    return out


def check(packer, rng, apps, placed, labels, ig=None, n_ig=1, label=""):
    driver, execn, off = placed
    names = ["node-%07d" % v for v in range(len(labels))]
    zone, nz = ref.intern_metric_zones(labels)
    a = dict(apps)
    a["off"] = off
    got = packer.placement_metrics(a, placed, zone, ig, n_ig)
    want = ref.literal_batch(driver, execn, off, apps["count"], names, labels, ig, apps.get("group"), rng)
    rows = ref.records_to_rows(got)
    want = np.asarray(want, np.int64).reshape(-1, 6)
    bad = np.nonzero((rows != want).any(axis=1))[0]
    assert len(bad) == 0, (label, bad[:5], rows[bad[:3]], want[bad[:3]])
    return got


def sub(apps):
    return {k: apps[k] for k in APP_COLS if k in apps}


# ---- the plain packers --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo,mode", [(TIGHTLY, INDEPENDENT), (EVENLY, INDEPENDENT), (MINFRAG, INDEPENDENT),
                                       (TIGHTLY, FIFO_REFERENCE), (EVENLY, FIFO_EXACT), (TIGHTLY, FIFO_EXACT)])
def test_plain_packers_on_synth_workloads(gangpack, packer, algo, mode):
    from k8s_spark_scheduler_b200 import synth
    rng = np.random.default_rng(100 + 3 * algo + mode)
    n, q = 10000, 100000 if mode == INDEPENDENT else 50000
    nodes = synth.make_nodes(n)
    apps = sub(synth.make_apps(q, da_sweep=mode != INDEPENDENT))
    eoff, eorder = synth.group_orders(nodes)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    placed = packer.pack_batch(apps, algo, mode)
    got = check(packer, rng, apps, placed, labels_of(rng, n), label=(algo, mode))
    assert (got["collocation"] >= 0).sum() > 100


# ---- the zone packers ---------------------------------------------------------------------------------------------------
def test_zone_results_and_fallback(gangpack, packer):
    rng = np.random.default_rng(7)
    n, Z, q = 1000, 3, 400
    avail = [rng.integers(4, 64, n).astype(np.int64) * 1000, rng.integers(16, 256, n).astype(np.int64) * G, np.zeros(n, np.int64)]
    sched = [a + 8000 for a in avail[:2]] + [np.zeros(n, np.int64)]
    zone = rng.integers(0, Z, n)
    zone[:Z] = np.arange(Z)
    dorder, eorder = rng.permutation(n).astype(np.int32), rng.permutation(n).astype(np.int32)
    zs = list(dict.fromkeys(int(zone[v]) for v in dorder))
    eo, do, eoff, doff = [], [], [0], [0]
    for z in zs:
        eo += [int(v) for v in eorder if zone[v] == z]
        do += [int(v) for v in dorder if zone[v] == z]
        eoff.append(len(eo)); doff.append(len(do))
    packer.set_snapshot(*avail, np.array(eo, np.int32), np.array(do, np.int32), np.array(eoff, np.int32), np.array(doff, np.int32))
    packer.set_schedulable(*sched)
    big = rng.random(q) < 0.3                  # 16-core executors: more than one zone holds, fewer than the cluster
    count = np.where(big, rng.integers(600, 1400, q), rng.integers(0, 24, q)).astype(np.int32)
    apps = {"drv_cpu": np.full(q, 1000, np.int64), "drv_mem": np.full(q, G, np.int64),
            "exe_cpu": np.where(big, 16000, rng.integers(1, 4, q) * 1000).astype(np.int64),
            "exe_mem": np.where(big, G, rng.integers(1, 8, q) * G).astype(np.int64), "count": count}
    # the metric zone is the failure-domain label: the packers' zones are not it
    labels = labels_of(rng, n, 5)
    for algo in (TIGHTLY, MINFRAG):
        _, drv, exe, off, _ = packer.pack_batch_zones(apps, algo)
        check(packer, rng, apps, (drv, exe, off), labels, label=("single-az", algo))
    zr, drv, exe, off, _ = packer.pack_batch_az_aware(apps, eorder, dorder, len(zs))
    assert ((zr == -1) & (drv >= 0)).any() and (zr >= 0).any()
    check(packer, rng, apps, (drv, exe, off), labels, label="az-aware")


# ---- every instance group's FIFO queue after gp_prepare_cluster_groups ------------------------------------------------------
@pytest.mark.parametrize("mode", [FIFO_REFERENCE, FIFO_EXACT])
def test_multi_group_drain(gangpack, packer, mode):
    from k8s_spark_scheduler_b200 import synth
    rng = np.random.default_rng(40 + mode)
    n, Gs, q = 4000, 16, 20000
    nodes = synth.make_nodes(n)
    ig = rng.integers(-1, Gs, n).astype(np.int32)
    alloc = [nodes["alloc_cpu"], nodes["alloc_mem"], nodes["alloc_gpu"]]
    used = [nodes["alloc_cpu"] - nodes["avail_cpu"], nodes["alloc_mem"] - nodes["avail_mem"], np.zeros(n, np.int64)]
    packer.prepare_cluster_groups(alloc, None, np.arange(n, dtype=np.int32), used, ig, Gs, orders=False)
    apps = sub(synth.make_apps(q, groups=Gs, da_sweep=True))
    placed = packer.pack_batch(apps, EVENLY if mode == FIFO_EXACT else TIGHTLY, mode)
    got = check(packer, rng, apps, placed, labels_of(rng, n), ig, Gs, label=("groups", mode))
    assert (got["collocation"] >= 0).sum() > 100


# ---- adversarial rows ---------------------------------------------------------------------------------------------------
def rows_case(rng, n, ks, driver_in=True):
    count = np.asarray(ks, np.int32)
    off = np.zeros(len(ks) + 1, np.int64)
    np.cumsum(count, out=off[1:])
    execn = rng.integers(0, n, int(off[-1])).astype(np.int32)
    driver = rng.integers(0, n, len(ks)).astype(np.int32)
    if driver_in:
        for i in range(0, len(ks), 2):
            if ks[i]:
                execn[off[i] + ks[i] // 2] = driver[i]
    return {"count": count}, (driver, execn, off)


def test_long_rows_and_every_node_its_own_zone(gangpack, packer):
    rng = np.random.default_rng(3)
    n = 10000
    ks = [0, 1, 2047, 2048, 2049, 5000, 70000, 3, 300000, 17]
    apps, placed = rows_case(rng, n, ks)
    check(packer, rng, apps, placed, labels_of(rng, n, 6), label="long rows")
    own = [{ref.LABEL_ZONE_FAILURE_DOMAIN: "z%d" % v} for v in range(n)]
    check(packer, rng, apps, placed, own, label="n_zones = n_nodes")
    ig = rng.integers(-1, 3, n).astype(np.int32)
    apps["group"] = rng.integers(0, 3, len(ks)).astype(np.int32)
    check(packer, rng, apps, placed, own, ig, 3, label="n_zones = n_nodes, instance groups")


def test_node_table_above_the_shared_memory_bitmap(gangpack, packer):
    """2 000 000 nodes: a bitmap of 250 KB does not fit in shared memory, the slices go to global scratch"""
    rng = np.random.default_rng(4)
    n = 2000000
    ks = [0, 5, 40, 3000, 100000, 2, 1]
    apps, placed = rows_case(rng, n, ks)
    shared = [{ref.LABEL_ZONE_FAILURE_DOMAIN: "zone-%d" % z} for z in range(7)]
    labels = [shared[v % 7] if v % 11 else {} for v in range(n)]
    check(packer, rng, apps, placed, labels, label="2M nodes")


# ---- the device form ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo,with_off", [(TIGHTLY, True), (TIGHTLY, False), (EVENLY, False), (MINFRAG, True)])
def test_device_form_reads_pack_batch_device_outputs(gangpack, packer, algo, with_off):
    import torch
    from k8s_spark_scheduler_b200 import synth
    native = gangpack.native
    rng = np.random.default_rng(9)
    n, q = 10000, 100000
    nodes = synth.make_nodes(n)
    apps = sub(synth.make_apps(q))
    off = synth.exec_offsets(apps["count"])
    eoff, eorder = synth.group_orders(nodes)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    dev = torch.device("cuda", 0)
    t = {k: torch.from_numpy(np.ascontiguousarray(apps[k])).to(dev) for k in ("drv_cpu", "drv_mem", "exe_cpu", "exe_mem", "count")}
    if with_off:
        t["off"] = torch.from_numpy(off).to(dev)
    d_drv = torch.full((q,), -7, dtype=torch.int32, device=dev)
    d_exe = torch.full((int(off[-1]),), -7, dtype=torch.int32, device=dev)
    packer.pack_batch_device(t, algo, INDEPENDENT, d_drv, d_exe)
    labels = labels_of(rng, n)
    zone, nz = ref.intern_metric_zones(labels)
    d_zone = torch.from_numpy(zone).to(dev)
    out = torch.zeros(native.PLACEMENT_DTYPE.itemsize * q, dtype=torch.uint8, device=dev)
    status = torch.full((1,), -1, dtype=torch.int32, device=dev)
    packer.placement_metrics_device(t, d_drv, d_exe, d_zone, out, nz, status=status)
    packer.synchronize()
    assert int(status.item()) == 0
    rec = out.cpu().numpy().view(native.PLACEMENT_DTYPE)
    placed = (d_drv.cpu().numpy(), d_exe.cpu().numpy(), off)
    host = packer.placement_metrics({"count": apps["count"], "off": off}, placed, zone)
    assert rec.tobytes() == host.tobytes()
    names = ["node-%07d" % v for v in range(n)]
    want = np.asarray(ref.literal_batch(*placed, apps["count"], names, labels, rng=rng), np.int64)
    assert np.array_equal(ref.records_to_rows(rec), want)


def test_device_form_with_instance_groups_and_refusal_status(gangpack, packer):
    import torch
    native = gangpack.native
    rng = np.random.default_rng(10)
    n = 3000
    apps, placed = rows_case(rng, n, [4, 0, 9000, 12, 1])
    apps["group"] = np.array([0, 1, 2, 1, 0], np.int32)
    ig = rng.integers(-1, 3, n).astype(np.int32)
    zone = (np.arange(n) % 5).astype(np.int32)
    dev = torch.device("cuda", 0)
    tt = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    t = {"count": tt(apps["count"]), "group": tt(apps["group"]), "off": tt(placed[2])}
    out = torch.zeros(native.PLACEMENT_DTYPE.itemsize * 5, dtype=torch.uint8, device=dev)
    status = torch.full((1,), -1, dtype=torch.int32, device=dev)
    packer.placement_metrics_device(t, tt(placed[0]), tt(placed[1]), tt(zone), out, 5, tt(ig), 3, status=status)
    packer.synchronize()
    assert int(status.item()) == 0
    host = packer.placement_metrics(dict(apps, off=placed[2]), placed, zone, ig, 3)
    assert out.cpu().numpy().view(native.PLACEMENT_DTYPE).tobytes() == host.tobytes()
    # refusals the device reports through the status word
    bad_exec = placed[1].copy(); bad_exec[3] = n
    for args, want in ((dict(exe=bad_exec), 1), (dict(zone=np.where(np.arange(n) == 7, 5, zone)), 1),
                       (dict(ig=np.where(np.arange(n) == 3, 3, ig)), 1), (dict(count=np.array([4, 0, 9000, -1, 1], np.int32)), 1),
                       (dict(cap=len(placed[1]) - 1), 5), (dict(count=np.array([4, 0, 9000, (1 << 24) + 1, 1], np.int32)), 6)):
        status.fill_(-1)
        t2 = dict(t)
        if "count" in args:
            t2["count"] = tt(args["count"])
        exe = tt(args.get("exe", placed[1]))
        if "cap" in args:
            exe = exe[:args["cap"]]
        packer.placement_metrics_device(t2, tt(placed[0]), exe, tt(args.get("zone", zone)), out, 5, tt(args.get("ig", ig)), 3,
                                        status=status)
        packer.synchronize()
        assert int(status.item()) == want, args.keys()
    # the state words are left zeroed: a valid call after the refusals succeeds
    status.fill_(-1)
    packer.placement_metrics_device(t, tt(placed[0]), tt(placed[1]), tt(zone), out, 5, tt(ig), 3, status=status)
    packer.synchronize()
    assert int(status.item()) == 0 and out.cpu().numpy().view(native.PLACEMENT_DTYPE).tobytes() == host.tobytes()


# ---- state and refusals -------------------------------------------------------------------------------------------------
def test_state_is_untouched(gangpack, packer):
    from k8s_spark_scheduler_b200 import synth
    rng = np.random.default_rng(11)
    n, q = 2000, 3000
    nodes = synth.make_nodes(n)
    apps = sub(synth.make_apps(q))
    eoff, eorder = synth.group_orders(nodes)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    placed = packer.pack_batch(apps, TIGHTLY, FIFO_EXACT)
    snap, stats = packer.get_snapshot(), packer.stats()
    check(packer, rng, apps, placed, labels_of(rng, n))
    assert all(np.array_equal(a, b) for a, b in zip(snap, packer.get_snapshot()))
    assert packer.stats() == stats
    # and no snapshot is needed
    fresh = gangpack.GangPacker()
    try:
        check(fresh, rng, apps, placed, labels_of(rng, n))
    finally:
        fresh.close()


def test_refusals(gangpack, packer):
    Err = gangpack.native.GangpackError
    rng = np.random.default_rng(12)
    n = 100
    apps, placed = rows_case(rng, n, [3, 0, 5])
    driver, execn, off = placed
    zone = (np.arange(n) % 4).astype(np.int32)
    a = dict(apps, off=off)

    def refused(status, fragment, **kw):
        args = dict(apps=a, placed=placed, metric_zone=zone)
        args.update(kw)
        with pytest.raises(Err) as e:
            packer.placement_metrics(**args)
        assert e.value.status == status and fragment in str(e.value), str(e.value)

    refused(1, "outside [0, n_nodes)", placed=(np.array([n, 1, 2], np.int32), execn, off))
    bad = execn.copy(); bad[4] = -3
    refused(1, "outside [0, n_nodes)", placed=(driver, bad, off))
    refused(1, "metric_zone outside", metric_zone=np.where(np.arange(n) == 50, -1, zone))
    refused(1, "metric_zone outside", metric_zone=zone, n_metric_zones=2)
    refused(1, "n_metric_zones above", n_metric_zones=n + 1)
    ig = (np.arange(n) % 2).astype(np.int32)
    refused(1, "instance_group outside", instance_group=np.where(np.arange(n) == 9, 2, ig), n_instance_groups=2)
    refused(1, "instance_group outside", apps=dict(a, group=np.array([0, 2, 1], np.int32)), instance_group=ig, n_instance_groups=2)
    refused(1, "n_instance_groups", instance_group=ig, n_instance_groups=0)
    refused(1, "negative exe_count", apps={"count": np.array([3, -1, 5], np.int32), "off": off})
    refused(5, "executor_nodes_cap", placed=(driver, execn[:-1], off))
    refused(6, "exe_count above 2^24", apps={"count": np.array([3, (1 << 24) + 1, 5], np.int32), "off": off})
    # a row that is not placed reads nothing: its offsets are not checked
    d2 = driver.copy(); d2[2] = -1
    got = packer.placement_metrics(a, (d2, execn[:-1], off), zone)
    assert tuple(got[2]) == ref.NOT_REPORTED
