"""Parity of the CUDA path (through the C ABI, libgangpack.so) against the CPU oracle: bit-exact
driver nodes and ExecutorNodes (contents AND order) on golden vectors, randomized edge-case
clusters, the synthetic bench workload, and all FIFO modes including the final snapshot."""
import numpy as np
import pytest

from helpers import (ALGO_ID, MODE_ID, assert_same_results, case_arrays, fifo_vs_closed, order_indices, random_apps,
                     random_cluster, res_aos)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def packer(gangpack):
    p = gangpack.GangPacker()
    yield p
    p.close()


def _oracle_batch(oracle, algo, mode, cpu, mem, gpu, drv_idx, exec_idx, apps, young=None):
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"])
    exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    blocked, dn, en, off, final = oracle.closed_batch(algo, mode, cpu, mem, gpu, drv_idx, exec_idx, drv, exe,
                                                      apps["count"], young, n_threads=8 if mode == 0 else 1)
    return blocked, (dn, en, off), final


def test_golden_pack_cases(golden, packer):
    for case in golden["pack_cases"]:
        names, cpu, mem, gpu = case_arrays(case["nodes"])
        packer.set_snapshot(cpu, mem, gpu, order_indices(case["exec_order"], names),
                            order_indices(case["driver_order"], names))
        app = case["app"]
        for algo, aid in ALGO_ID.items():
            ok, d, ex = packer.pack_one(aid, app["drv"], app["exe"], app["count"])
            exp = case["expect"][algo]
            assert ok == exp["fit"], (case["id"], algo)
            if ok:
                assert names[d] == exp["driver"], (case["id"], algo)
                assert [names[i] for i in ex] == exp["executors"], (case["id"], algo)
        c2, m2, g2 = packer.get_snapshot()   # independent packs never mutate the snapshot
        assert np.array_equal(c2, cpu) and np.array_equal(m2, mem) and np.array_equal(g2, gpu)


def test_golden_fifo_cases(golden, packer):
    for case in golden["fifo_cases"]:
        names, cpu, mem, gpu = case_arrays(case["nodes"])
        idx = np.arange(len(names), dtype=np.int32)
        packer.set_snapshot(cpu, mem, gpu, idx, idx)
        apps = case["apps"]
        a = {"drv_cpu": [x["drv"][0] for x in apps], "drv_mem": [x["drv"][1] for x in apps],
             "drv_gpu": [x["drv"][2] for x in apps], "exe_cpu": [x["exe"][0] for x in apps],
             "exe_mem": [x["exe"][1] for x in apps], "exe_gpu": [x["exe"][2] for x in apps],
             "count": [x["count"] for x in apps], "young": [1 if x.get("young") else 0 for x in apps]}
        dn, en, off = packer.pack_batch(a, ALGO_ID[case["algo"]], MODE_ID[case["mode"]])
        exp = case["expect"]
        for i, r in enumerate(exp["results"]):
            if r["driver"] == "unevaluated":
                assert dn[i] == -2, case["id"]
            elif r["driver"] is None:
                assert dn[i] == -1, case["id"]
            else:
                assert names[dn[i]] == r["driver"], case["id"]
                assert [names[j] for j in en[off[i]:off[i + 1]]] == r["executors"], case["id"]
        fc, fm, fg = packer.get_snapshot()
        for j, f in enumerate(exp["final_available"]):
            assert (fc[j], fm[j], fg[j]) == (f["cpu"], f["mem"], f["gpu"]), case["id"]


@pytest.mark.parametrize("seed", range(10))
def test_random_independent(oracle, packer, seed):
    rng = np.random.default_rng(3000 + seed)
    for trial in range(5):
        n = int(rng.integers(1, 200))
        cpu, mem, gpu = random_cluster(rng, n, tight=bool(trial % 2), gpus=bool(seed % 2), negative=bool(seed % 3 == 0))
        perm = rng.permutation(n)
        exec_idx = perm[rng.random(n) < 0.85].astype(np.int32)
        drv_idx = rng.permutation(n)[: max(1, int(n * rng.uniform(0.3, 1.0)))].astype(np.int32)
        apps = random_apps(rng, 200, gpus=bool(seed % 2), zero_dims=bool(seed % 4 == 1), big_counts=bool(seed % 4 == 2))
        packer.set_snapshot(cpu, mem, gpu, exec_idx, drv_idx)
        for algo in (0, 1):
            _, want, _ = _oracle_batch(oracle, algo, 0, cpu, mem, gpu, drv_idx, exec_idx, apps)
            got = packer.pack_batch(apps, algo, 0)
            assert_same_results(got, want, f"seed {seed} trial {trial} algo {algo}")


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("mode", [1, 2])
def test_random_fifo(oracle, packer, seed, mode):
    rng = np.random.default_rng(4000 + seed)
    for trial in range(4):
        n = int(rng.integers(2, 300))
        cpu, mem, gpu = random_cluster(rng, n, gpus=bool(seed % 2))
        perm = rng.permutation(n)
        exec_idx = perm[rng.random(n) < 0.9].astype(np.int32)
        drv_idx = rng.permutation(n)[: max(1, int(n * rng.uniform(0.3, 1.0)))].astype(np.int32)
        q = 300
        apps = random_apps(rng, q, gpus=bool(seed % 2), zero_dims=bool(seed % 3 == 1), big_counts=bool(trial == 3))
        young = (rng.random(q) < (0.9 if trial % 2 else 0.2)).astype(np.uint8)
        apps["young"] = young
        for algo in (0, 1):
            packer.set_snapshot(cpu, mem, gpu, exec_idx, drv_idx)
            blocked, want, final = _oracle_batch(oracle, algo, mode, cpu, mem, gpu, drv_idx, exec_idx, apps, young)
            got = packer.pack_batch(apps, algo, mode)
            assert_same_results(got, want, f"seed {seed} trial {trial} algo {algo} mode {mode}")
            fc, fm, fg = packer.get_snapshot()
            assert np.array_equal(fc, final[0]) and np.array_equal(fm, final[1]) and np.array_equal(fg, final[2])


def test_awkward_divisors(oracle, packer):
    """Exercise every division path of cap_dim: power-of-two, magic (odd < 2^32), slow (odd >= 2^32),
    shifted numerators above 2^32, 1-byte requests (reference tests use mem '1')."""
    rng = np.random.default_rng(77)
    n = 64
    cpu = rng.integers(0, 1 << 40, n).astype(np.int64)
    mem = rng.integers(0, 1 << 45, n).astype(np.int64)
    gpu = np.zeros(n, np.int64)
    idx = np.arange(n, dtype=np.int32)
    exe_mem = np.array([1, 3, 1 << 20, (1 << 20) * 3, (1 << 33) + 1, (1 << 34) + 2, 7 << 31, 12345678901, 1 << 44, 5], np.int64)
    q = len(exe_mem) * 4
    apps = {
        "drv_cpu": np.zeros(q, np.int64), "drv_mem": rng.integers(0, 1 << 30, q).astype(np.int64), "drv_gpu": np.zeros(q, np.int64),
        "exe_cpu": np.tile(np.array([1, 1000, 4097, (1 << 35) + 7], np.int64), len(exe_mem)),
        "exe_mem": np.repeat(exe_mem, 4), "exe_gpu": np.zeros(q, np.int64),
        "count": rng.integers(1, 3000, q).astype(np.int32),
    }
    packer.set_snapshot(cpu, mem, gpu, idx, idx)
    for algo in (0, 1):
        _, want, _ = _oracle_batch(oracle, algo, 0, cpu, mem, gpu, idx, idx, apps)
        got = packer.pack_batch(apps, algo, 0)
        assert_same_results(got, want, f"awkward algo {algo}")


def test_multi_group(oracle, packer):
    """Instance groups: disjoint node sets with their own orders; FIFO queues are per group
    (sparkpods.go:61, resource.go:292-295) and must equal the oracle run per group."""
    import k8s_spark_scheduler_b200.synth as synth
    G = 5
    nodes = synth.make_nodes(700, groups=G)
    apps = synth.make_apps(900, groups=G, young_frac=0.1)
    eoff, eorder = synth.group_orders(nodes)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group", "young")}
    for algo in (0, 1):
        for mode in (0, 1, 2):
            packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
            dn, en, off = packer.pack_batch(a, algo, mode)
            for g in range(G):
                sel = np.nonzero(apps["group"] == g)[0]
                sub = {k: np.asarray(v)[sel] for k, v in a.items()}
                order = eorder[eoff[g]:eoff[g + 1]]
                _, want, _ = _oracle_batch(oracle, algo, mode, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"],
                                           order, order, sub, sub["young"] if mode else None)
                wd, we, woff = want
                assert np.array_equal(dn[sel], wd), (algo, mode, g)
                for j, i in enumerate(sel):
                    if wd[j] >= 0:
                        assert np.array_equal(en[off[i]:off[i + 1]], we[woff[j]:woff[j + 1]]), (algo, mode, g, i)


def test_synthetic_bench_workload_sample(oracle, packer):
    """BASELINE configs[1]/[2] shape (10k nodes) on a 4k-app sample: bit-exact vs the oracle."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000)
    apps = synth.make_apps(4000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    for algo in (0, 1):
        _, want, _ = _oracle_batch(oracle, algo, 0, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order, a)
        got = packer.pack_batch(a, algo, 0)
        assert_same_results(got, want, f"synthetic algo {algo}")
        assert (got[0] >= 0).all()


def test_full_size_properties(packer):
    """BASELINE full size (10k nodes x 100k apps): size-independent properties instead of the oracle:
    every placement respects capacity, ExecutorNodes has the algorithm's shape, and the batch equals
    the concatenation of two half batches (independence)."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000)
    apps = synth.make_apps(100000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    rank = np.empty(10000, np.int64); rank[order] = np.arange(10000)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    for algo in (0, 1):
        dn, en, off = packer.pack_batch(a, algo, 0)
        assert (dn >= 0).all()
        h = 50000
        first = packer.pack_batch({k: v[:h] for k, v in a.items()}, algo, 0)
        second = packer.pack_batch({k: v[h:] for k, v in a.items()}, algo, 0)
        assert np.array_equal(dn, np.concatenate([first[0], second[0]]))
        assert np.array_equal(en, np.concatenate([first[1], second[1]]))
        # capacity: per app, driver + executors on each node fit the node
        app_of = np.repeat(np.arange(100000), apps["count"])
        key = app_of * 10000 + en
        uniq, cnt = np.unique(key, return_counts=True)
        ua, un = uniq // 10000, uniq % 10000
        on_driver = (dn[ua] == un)
        need_cpu = cnt * apps["exe_cpu"][ua] + on_driver * apps["drv_cpu"][ua]
        need_mem = cnt * apps["exe_mem"][ua] + on_driver * apps["drv_mem"][ua]
        assert (need_cpu <= nodes["avail_cpu"][un]).all() and (need_mem <= nodes["avail_mem"][un]).all()
        assert (apps["drv_cpu"] <= nodes["avail_cpu"][dn]).all() and (apps["drv_mem"] <= nodes["avail_mem"][dn]).all()
        r = rank[en]
        same_app = app_of[1:] == app_of[:-1]
        if algo == 0:   # node-major: priority rank is non-decreasing inside an app
            assert (r[1:][same_app] >= r[:-1][same_app]).all()
        else:           # round-major with one round here: strictly increasing ranks unless a new round starts
            assert ((r[1:][same_app] > r[:-1][same_app]) | (cnt.max() > 1)).all()


def test_error_paths(packer):
    Gi = 1 << 30
    idx = np.arange(2, dtype=np.int32)
    packer.set_snapshot([8000, 8000], [8 * Gi, 8 * Gi], [0, 0], idx, idx)
    base = {"drv_cpu": [1000], "drv_mem": [Gi], "drv_gpu": [0], "exe_cpu": [1000], "exe_mem": [Gi], "exe_gpu": [0], "count": [1]}
    from k8s_spark_scheduler_b200 import GangpackError
    with pytest.raises(GangpackError) as e:
        packer.pack_batch({**base, "exe_cpu": [-1]}, 0, 0)
    assert e.value.status == 1
    with pytest.raises(GangpackError) as e:
        packer.pack_batch({**base, "exe_mem": [1 << 62]}, 0, 0)
    assert e.value.status == 6
    with pytest.raises(GangpackError) as e:
        packer.pack_batch({**base, "group": [3]}, 0, 0)
    assert e.value.status == 1
    with pytest.raises(GangpackError) as e:
        packer.set_snapshot([1, 2], [1, 2], [0, 0], np.array([0, 0], np.int32), idx)   # duplicate node in an order
    assert e.value.status == 1
    # the context is still usable after errors
    dn, en, off = packer.pack_batch(base, 0, 0)
    assert dn[0] == 0 and en[0] == 0
    # empty batch
    dn, en, off = packer.pack_batch({k: [] for k in base}, 0, 0)
    assert len(dn) == 0


def test_pinned_host_paths(oracle, packer):
    """Every host-buffer route of gp_pack_batch gives the same bits: pageable (DMA staging), mapped pinned small
    batch (inputs read in place, results written in place), pinned equally spaced columns (one 2-D DMA per
    chunk, pipelined chunks) and pinned scattered columns."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(3000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    keys = ("drv_cpu", "drv_mem", "exe_cpu", "exe_mem", "drv_gpu", "exe_gpu")
    for q in (1500, 70000):
        apps = synth.make_apps(q, gpu_variant=True)
        a = {k: apps[k] for k in keys + ("count",)}
        ref = packer.pack_batch(a, 0, 0)                                   # pageable numpy arrays
        if q == 1500:
            _, want, _ = _oracle_batch(oracle, 0, 0, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order, a)
            assert_same_results(ref, want, "pageable")
        total = int(ref[2][-1])
        cols = packer.pinned_columns(q, keys)                              # one block, equally spaced
        for k in keys:
            cols[k][:] = a[k]
        cols["count"] = packer.pinned(q, np.int32); cols["count"][:] = a["count"]
        cols["off"] = packer.pinned(q + 1, np.int64); cols["off"][:] = ref[2]
        od = packer.pinned(q, np.int32); oe = packer.pinned(max(total, 1), np.int32)
        od[:] = -7; oe[:] = -7
        got = packer.pack_batch(cols, 0, 0, out=(od, oe))
        assert_same_results(got, ref, f"pinned columns q={q}")
        scattered = {k: packer.pinned(q, np.int64) for k in keys}          # separate allocations
        for k in keys:
            scattered[k][:] = a[k]
        scattered["count"] = cols["count"]; scattered["off"] = cols["off"]
        od[:] = -7; oe[:] = -7
        got = packer.pack_batch(scattered, 1, 0, out=(od, oe))
        ref1 = packer.pack_batch(a, 1, 0)
        assert_same_results(got, ref1, f"pinned scattered q={q}")
        # drop the all-or-nothing gpu columns one at a time (NULL = 0 semantics)
        no_gpu = {k: v for k, v in cols.items() if k not in ("drv_gpu", "exe_gpu")}
        a0 = dict(a); a0["drv_gpu"] = np.zeros(q, np.int64); a0["exe_gpu"] = np.zeros(q, np.int64)
        assert_same_results(packer.pack_batch(no_gpu, 0, 0, out=(od, oe)), packer.pack_batch(a0, 0, 0), f"NULL gpu columns q={q}")


def test_pinned_host_paths_dma_route():
    """Same test with mapped-memory access disabled: every buffer takes the (2-D) DMA staging route."""
    import os, subprocess, sys
    env = dict(os.environ, GANGPACK_ZERO_COPY="0")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_gpu_parity.py"), "-m", "gpu", "-q", "-x",
                        "-k", "test_pinned_host_paths and not dma_route"], env=env, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]


def test_large_cluster_and_big_fifo_group(oracle, packer):
    """BASELINE configs[4] shape (50k nodes) on a sample, and a FIFO group larger than the shared-memory
    staging area (slots beyond it are served from global memory by the same kernel)."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(50000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    apps = synth.make_apps(3000)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    for algo in (0, 1):
        _, want, _ = _oracle_batch(oracle, algo, 0, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order, a)
        assert_same_results(packer.pack_batch(a, algo, 0), want, f"50k nodes algo {algo}")
    # FIFO over 14 000 nodes (> 11 776 staged slots), queue long enough to reach deep into the order
    n = 14000
    sub = {k: v[:n] for k, v in nodes.items() if hasattr(v, "__len__")}
    order = synth.priority_order(sub["avail_cpu"], sub["avail_mem"])
    big = synth.make_apps(6000, seed=77)
    a = {k: big[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    a["exe_cpu"] = a["exe_cpu"] * 4; a["count"] = np.minimum(a["count"] * 4, 100).astype(np.int32)   # hungry apps: fill the cluster
    young = (np.arange(6000) % 3 == 0).astype(np.uint8)
    a["young"] = young
    for algo in (0, 1):
        for mode in (1, 2):
            packer.set_snapshot(sub["avail_cpu"], sub["avail_mem"], sub["avail_gpu"], order, order)
            blocked, want, final = _oracle_batch(oracle, algo, mode, sub["avail_cpu"], sub["avail_mem"], sub["avail_gpu"], order, order, a, young)
            got = packer.pack_batch(a, algo, mode)
            assert_same_results(got, want, f"big fifo algo {algo} mode {mode}")
            fc, fm, fg = packer.get_snapshot()
            assert np.array_equal(fc, final[0]) and np.array_equal(fm, final[1])


def test_degenerate_groups(oracle, packer):
    """Groups with no executor candidates / no driver candidates, and apps pointing at them."""
    Gi = 1 << 30
    cpu = np.array([8000, 8000, 8000, 8000], np.int64); mem = np.full(4, 16 * Gi, np.int64); gpu = np.zeros(4, np.int64)
    # group 0: nodes 0,1 both orders; group 1: drivers only (node 2); group 2: executors only (node 3); group 3: empty
    eoff = np.array([0, 2, 2, 3, 3], np.int32); eorder = np.array([0, 1, 3], np.int32)
    doff = np.array([0, 2, 3, 3, 3], np.int32); dorder = np.array([0, 1, 2], np.int32)
    packer.set_snapshot(cpu, mem, gpu, eorder, dorder, eoff, doff)
    apps = {"drv_cpu": [1000] * 8, "drv_mem": [Gi] * 8, "drv_gpu": [0] * 8, "exe_cpu": [2000] * 8, "exe_mem": [4 * Gi] * 8,
            "exe_gpu": [0] * 8, "count": [2, 0, 2, 0, 2, 0, 2, 0], "group": [0, 0, 1, 1, 2, 2, 3, 3]}
    for algo in (0, 1):
        for mode in (0, 1, 2):
            packer.set_snapshot(cpu, mem, gpu, eorder, dorder, eoff, doff)
            young = np.ones(8, np.uint8)
            dn, en, off = packer.pack_batch({**apps, "young": young}, algo, mode)
            assert dn[0] == 0 and dn[1] >= 0          # group 0 works; count 0 needs only a driver
            assert dn[2] == -1 and dn[3] == 2         # group 1: no executor candidates: count 2 fails, count 0 fits on node 2
            assert dn[4] == -1 and dn[5] == -1        # group 2: no driver candidates
            assert dn[6] == -1 and dn[7] == -1        # group 3: empty


def test_device_resident_api(oracle, packer):
    """gp_set_snapshot_device / gp_pack_batch_device (what bench.py's `value` path and the NCCL path use)."""
    import torch
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(2000, groups=3)
    apps = synth.make_apps(5000, groups=3)
    eoff, eorder = synth.group_orders(nodes)
    dev = torch.device("cuda", 0)
    t = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(dt).to(dev)
    tn = [t(nodes["avail_cpu"], torch.int64), t(nodes["avail_mem"], torch.int64), t(nodes["avail_gpu"], torch.int64),
          t(eoff, torch.int32), t(eorder, torch.int32)]
    off = synth.exec_offsets(apps["count"])
    ta = {k: t(apps[k], torch.int64) for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu")}
    ta["count"] = t(apps["count"], torch.int32); ta["group"] = t(apps["group"], torch.int32); ta["off"] = t(off, torch.int64)
    d_driver = torch.full((5000,), -9, dtype=torch.int32, device=dev)
    d_exec = torch.full((int(off[-1]),), -9, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group")}
    for algo in (0, 1):
        packer.set_snapshot_device(tn[0], tn[1], tn[2], tn[3], tn[4], tn[3], tn[4])
        packer.pack_batch_device(ta, algo, 0, d_driver, d_exec)
        packer.synchronize()
        st = packer.stats()
        assert st["nodes_scanned"] > 0 and st["pack_kernel_ns"] > 0
        packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
        want = packer.pack_batch(a, algo, 0)
        assert_same_results((d_driver.cpu().numpy(), d_exec.cpu().numpy(), off), want, f"device api algo {algo}")


@pytest.mark.parametrize("mode", [1, 2])
def test_fifo_full_size_conservation(oracle, packer, mode):
    """BASELINE configs[1] in FIFO mode at full size (10k nodes x 10k apps): size-independent properties.
    (i) conservation: initial - final availability equals the usage recomputed from the emitted placements under
    the mode's accounting (reference: each distinct executor node one executor, driver node charged the driver
    only if it hosts no executor -- EXT/sparkpods.go:139-146; exact: every pod); (ii) after the first blocking
    application nothing is evaluated; (iii) every placement respected the availability at its turn (no node
    ever goes below its running balance by more than the accounting allows); (iv) every one of the 10 000 decisions and
    the final snapshot equal the closed-form oracle's."""
    import k8s_spark_scheduler_b200.synth as synth
    N, Q = 10000, 10000
    nodes = synth.make_nodes(N)
    apps = synth.make_apps(Q)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    young = (np.arange(Q) % 7 == 0).astype(np.uint8)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    a["young"] = young
    for algo in (0, 1):
        packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
        dn, en, off = packer.pack_batch(a, algo, mode)
        fc, fm, _ = packer.get_snapshot()
        fits = dn >= 0
        # (ii) block semantics
        nofit_old = np.nonzero((dn == -1) & (young == 0))[0]
        if nofit_old.size:
            b = nofit_old[0]
            assert (dn[b + 1:] == -2).all() and (dn[:b] != -2).all()
        else:
            assert (dn != -2).all()
        # (i) conservation
        app_of = np.repeat(np.arange(Q), apps["count"])
        keep = fits[app_of]
        ea, eno = app_of[keep], en[:len(app_of)][keep]
        use_cpu = np.zeros(N, np.int64); use_mem = np.zeros(N, np.int64)
        if mode == 2:
            np.add.at(use_cpu, eno, apps["exe_cpu"][ea]); np.add.at(use_mem, eno, apps["exe_mem"][ea])
            np.add.at(use_cpu, dn[fits], apps["drv_cpu"][fits]); np.add.at(use_mem, dn[fits], apps["drv_mem"][fits])
        else:
            key = np.unique(ea.astype(np.int64) * N + eno)
            ua, un = key // N, key % N
            np.add.at(use_cpu, un, apps["exe_cpu"][ua]); np.add.at(use_mem, un, apps["exe_mem"][ua])
            hosted = np.zeros(Q, bool)
            hosted[ua[dn[ua] == un]] = True
            drv_only = fits & ~hosted
            np.add.at(use_cpu, dn[drv_only], apps["drv_cpu"][drv_only]); np.add.at(use_mem, dn[drv_only], apps["drv_mem"][drv_only])
        assert np.array_equal(nodes["avail_cpu"] - use_cpu, fc), (algo, mode)
        assert np.array_equal(nodes["avail_mem"] - use_mem, fm), (algo, mode)
        assert fits.sum() > 1000
        # (iv) bit-exact against the oracle
        final = fifo_vs_closed(oracle, algo, mode, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order,
                               [0, N], [0, N], a, (dn, en, off), f"fifo full size algo {algo} mode {mode}")
        fg = packer.get_snapshot()[2]
        assert np.array_equal(fc, final[0]) and np.array_equal(fm, final[1]) and np.array_equal(fg, final[2]), (algo, mode)


@pytest.mark.parametrize("mode", [1, 2])
def test_fifo_da_50k_vs_oracle(oracle, packer, mode):
    """bench.py's fifo-da-50k shape (BASELINE configs[3]: 10k nodes in 16 instance groups, 50 000 queued drivers of a
    dynamic-allocation sweep), every decision and the final snapshot against the closed form, group by group."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000, groups=16)
    apps = synth.make_apps(50000, groups=16, da_sweep=True, young_frac=0.05)
    eoff, eorder = synth.group_orders(nodes)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group", "young")}
    for algo in (0, 1):
        packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
        got = packer.pack_batch(a, algo, mode)
        final = fifo_vs_closed(oracle, algo, mode, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder,
                               eoff, eoff, a, got, f"fifo-da-50k algo {algo} mode {mode}")
        fc, fm, fg = packer.get_snapshot()
        assert np.array_equal(fc, final[0]) and np.array_equal(fm, final[1]) and np.array_equal(fg, final[2]), (algo, mode)
        assert (got[0] >= 0).sum() > 10000


def _potential_nodes_inputs(names, zones):
    zid, seen = [], {}
    for n in names:
        z = zones.get(n, "default")
        zid.append(seen.setdefault(z, len(seen)))           # dense ids in first-seen order
    order = sorted(range(len(names)), key=lambda i: names[i])
    rank = np.empty(len(names), np.int32); rank[order] = np.arange(len(names))
    return np.array(zid, np.int32), max(len(seen), 1), rank


def test_potential_nodes_goldens(golden, packer):
    """internal/sort/nodesorting_test.go:98-252 through the device implementation of PotentialNodes."""
    for case in golden["sort_cases"]:
        names, cpu, mem, gpu = case_arrays(case["nodes"])
        zid, nz, rank = _potential_nodes_inputs(names, case["zones"])
        d, e = packer.potential_nodes(cpu, mem, zid, nz, rank)
        assert [names[i] for i in d] == case["expect_priority_order"], case["id"]
        assert [names[i] for i in e] == case["expect_priority_order"], case["id"]
    for case in golden["label_cases"]:
        names = case["input"]
        n = len(names)
        zid, nz, rank = _potential_nodes_inputs(names, {})
        lr = np.array([case["rank"].get(nm, -1) for nm in names], np.int32)
        d, e = packer.potential_nodes(np.ones(n, np.int64), np.arange(1, n + 1, dtype=np.int64), zid, nz, rank,
                                      driver_label_rank=lr, executor_label_rank=lr)
        assert [names[i] for i in d] == case["expect"] and [names[i] for i in e] == case["expect"], case["id"]


@pytest.mark.parametrize("seed", range(6))
def test_potential_nodes_random(oracle, packer, seed):
    """Device PotentialNodes == the literal oracle on random multi-zone clusters with heavy (memory, cpu) ties,
    candidate subsets, unschedulable / not-ready nodes and label priorities (inputs avoid the ties the reference
    itself leaves undefined: gpu is constant)."""
    rng = np.random.default_rng(5000 + seed)
    for n in (1, 2, 37, 700, 5000):
        names = ["node-%05d" % int(x) for x in rng.permutation(n * 3)[:n]]
        cpu = rng.integers(0, 6, n) * 1000
        mem = rng.integers(0, 5, n) * (1 << 30)
        zones = {nm: "zone-%d" % rng.integers(0, 4) for nm in names} if seed % 2 else {}
        unsched = (rng.random(n) < 0.1).astype(np.uint8)
        ready = (rng.random(n) < 0.9).astype(np.uint8)
        cand_mask = (rng.random(n) < 0.6).astype(np.uint8)
        lr_d = rng.integers(-1, 3, n).astype(np.int32) if seed % 3 == 0 else None
        lr_e = rng.integers(-1, 2, n).astype(np.int32) if seed % 3 != 1 else None
        cl = oracle.Cluster(names, cpu, mem, np.zeros(n, np.int64), zone=[zones.get(nm, "default") for nm in names],
                            unschedulable=unsched, ready=ready)
        wd, we = cl.potential_nodes([nm for nm, m in zip(names, cand_mask) if m], lr_d, lr_e)
        zid, nz, rank = _potential_nodes_inputs(names, zones)
        d, e = packer.potential_nodes(cpu, mem, zid, nz, rank, cand_mask, unsched, ready, lr_d, lr_e)
        assert [names[i] for i in d] == wd, (seed, n)
        assert [names[i] for i in e] == we, (seed, n)


def test_potential_nodes_feeds_the_packer(oracle, packer):
    """sort on the device -> snapshot -> pack == the host-sorted reference flow (synthetic 10k-node cluster)."""
    import k8s_spark_scheduler_b200.synth as synth
    nodes = synth.make_nodes(10000)
    host_order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    d, e = packer.potential_nodes(nodes["avail_cpu"], nodes["avail_mem"])
    assert np.array_equal(d, host_order) and np.array_equal(e, host_order)
    apps = synth.make_apps(2000)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], e, d)
    _, want, _ = _oracle_batch(oracle, 0, 0, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], host_order, host_order, a)
    assert_same_results(packer.pack_batch(a, 0, 0), want, "device-sorted orders")


def test_build_availability(oracle, packer):
    """f2: reservations (hard + soft) and overhead -> available / schedulable on the device == literal oracle."""
    rng = np.random.default_rng(11)
    for n, R in ((1, 0), (50, 400), (10000, 250000)):
        names = ["node-%05d" % i for i in range(n)]
        alloc = [rng.integers(1, 97, n) * 1000, rng.integers(1, 385, n) * (1 << 30), rng.integers(0, 9, n)]
        over = [rng.integers(0, 3, n) * 250, rng.integers(0, 4, n) * (1 << 28), np.zeros(n, np.int64)]
        rnode = rng.integers(-1, n, R).astype(np.int32)          # -1: reservation on a node that left the cluster
        res = [rng.integers(0, 8, R) * 500, rng.integers(0, 16, R) * (1 << 29), rng.integers(0, 2, R)]
        av, sc = packer.build_availability(alloc, over, rnode, res)
        rn = [names[i] if i >= 0 else "gone" for i in rnode]
        wav, wsc = oracle.node_scheduling_metadata(names, alloc, over, rn, res)
        for d in range(3):
            assert np.array_equal(av[d], wav[d]) and np.array_equal(sc[d], wsc[d]), (n, R, d)
        av2, _ = packer.build_availability(alloc, None, rnode, res)      # no overhead arrays
        assert np.array_equal(av2[0], av[0] + over[0])


def test_prepare_cluster_chain(oracle, packer):
    """gp_prepare_cluster (reservations -> availability -> orders -> snapshot, all on the device) followed by a
    FIFO batch == the same steps through the separate entries == the CPU oracle end to end."""
    rng = np.random.default_rng(21)
    n, R, q = 3000, 40000, 800
    names = ["node-%05d" % int(x) for x in rng.permutation(n * 2)[:n]]
    alloc = [rng.integers(8, 97, n) * 1000, rng.integers(32, 385, n) * (1 << 30), np.zeros(n, np.int64)]
    over = [rng.integers(0, 3, n) * 250, rng.integers(0, 4, n) * (1 << 28), np.zeros(n, np.int64)]
    rnode = rng.integers(-1, n, R).astype(np.int32)
    res = [rng.integers(0, 6, R) * 500, rng.integers(0, 12, R) * (1 << 29), np.zeros(R, np.int64)]
    zones = {nm: "zone-%d" % rng.integers(0, 3) for nm in names}
    zid, nz, rank = _potential_nodes_inputs(names, zones)
    unsched = (rng.random(n) < 0.05).astype(np.uint8); ready = (rng.random(n) < 0.95).astype(np.uint8)
    cand = (rng.random(n) < 0.8).astype(np.uint8)
    import k8s_spark_scheduler_b200.synth as synth
    apps = synth.make_apps(q, seed=5)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    a["young"] = (np.arange(q) % 5 == 0).astype(np.uint8)
    # chained on the device
    nd, ne = packer.prepare_cluster(alloc, over, rnode, res, zid, nz, rank, cand, unsched, ready)
    got = packer.pack_batch(a, 0, 1)
    snap = packer.get_snapshot()
    # the same through the separate entries
    av, _ = packer.build_availability(alloc, over, rnode, res)
    d, e = packer.potential_nodes(av[0], av[1], zid, nz, rank, cand, unsched, ready)
    assert (nd, ne) == (len(d), len(e))
    packer.set_snapshot(av[0], av[1], av[2], e, d)
    want = packer.pack_batch(a, 0, 1)
    assert_same_results(got, want, "chained vs separate")
    for x, y in zip(snap, packer.get_snapshot()):
        assert np.array_equal(x, y)
    # and the CPU oracle end to end (string-keyed)
    rn = [names[i] if i >= 0 else "gone" for i in rnode]
    wav, _ = oracle.node_scheduling_metadata(names, alloc, over, rn, res)
    cl = oracle.Cluster(names, wav[0], wav[1], wav[2], zone=[zones[nm] for nm in names], unschedulable=unsched, ready=ready)
    wd, we = cl.potential_nodes([nm for nm, m in zip(names, cand) if m])
    drv = res_aos(a["drv_cpu"], a["drv_mem"], a["drv_gpu"]); exe = res_aos(a["exe_cpu"], a["exe_mem"], a["exe_gpu"])
    _, od, oe, ooff = cl.fifo(0, 1, drv, exe, a["count"], a["young"], wd, we)
    assert_same_results(got, (od, oe, ooff), "device pipeline vs literal oracle pipeline")


# ---------------------------------------------------------------------------------------------------------------
# minimal-fragmentation (SURVEY §8f row f3): device algo 2 == oracle algo 4 (LIB/binpack/minimal_fragmentation.go)
# ---------------------------------------------------------------------------------------------------------------
MF_DEV, MF_ORC = 2, 4


def test_minfrag_doc_examples(packer):
    """capacities a1 b1 c3 d5 e5 f17 (minimal_fragmentation.go:43-58); the count-19 line follows the code, not the comment"""
    names = ["a", "b", "c", "d", "e", "f", "drv"]
    cpu = np.array([1000, 1000, 3000, 5000, 5000, 17000, 500], np.int64)
    mem = np.full(7, 1 << 40, np.int64)
    packer.set_snapshot(cpu, mem, np.zeros(7, np.int64), np.arange(6, dtype=np.int32), np.array([6], np.int32))
    for count, expected in [(11, ["d"] * 5 + ["e"] * 5 + ["a"]), (6, ["d"] * 5 + ["a"]),
                            (15, ["d"] * 5 + ["e"] * 5 + ["c"] * 3 + ["a", "b"]), (17, ["f"] * 17),
                            (19, ["f"] * 17 + ["c", "c"]), (32, ["f"] * 17 + ["d"] * 5 + ["e"] * 5 + ["c"] * 3 + ["a", "b"]),
                            (0, [])]:
        ok, d, ex = packer.pack_one(MF_DEV, (500, 1, 0), (1000, 1, 0), count)
        assert ok and names[d] == "drv" and [names[i] for i in ex] == expected, count
    ok, _, _ = packer.pack_one(MF_DEV, (500, 1, 0), (1000, 1, 0), 33)
    assert not ok


def test_golden_minfrag_cases(golden, packer):
    for case in golden["minfrag_cases"]:
        names, cpu, mem, gpu = case_arrays(case["nodes"])
        packer.set_snapshot(cpu, mem, gpu, order_indices(case["exec_order"], names), order_indices(case["driver_order"], names))
        app, exp = case["app"], case["expect"]
        ok, d, ex = packer.pack_one(MF_DEV, app["drv"], app["exe"], app["count"])
        assert ok == exp["fit"], case["id"]
        if ok:
            assert names[d] == exp["driver"] and [names[i] for i in ex] == exp["executors"], case["id"]


@pytest.mark.parametrize("seed", range(10))
def test_minfrag_random(oracle, packer, seed):
    rng = np.random.default_rng(8000 + seed)
    for trial in range(5):
        n = int(rng.integers(1, 300))
        cpu, mem, gpu = random_cluster(rng, n, tight=bool(trial % 2), gpus=bool(seed % 2), negative=bool(seed % 3 == 0))
        perm = rng.permutation(n)
        exec_idx = perm[rng.random(n) < 0.85].astype(np.int32)
        drv_idx = rng.permutation(n)[: max(1, int(n * rng.uniform(0.3, 1.0)))].astype(np.int32)
        apps = random_apps(rng, 300, gpus=bool(seed % 2), zero_dims=bool(seed % 4 == 1), big_counts=bool(seed % 4 >= 2))
        packer.set_snapshot(cpu, mem, gpu, exec_idx, drv_idx)
        _, want, _ = _oracle_batch(oracle, MF_ORC, 0, cpu, mem, gpu, drv_idx, exec_idx, apps)
        got = packer.pack_batch(apps, MF_DEV, 0)
        assert_same_results(got, want, f"minfrag seed {seed} trial {trial}")


@pytest.mark.parametrize("seed", range(8))
def test_minfrag_dense_ties(oracle, packer, seed):
    """small capacities with many equal values, counts spread over [0, total + 3], every-dimension-zero executors
    (capacity math.MaxInt: the target computation wraps), consumed lists longer than one warp"""
    rng = np.random.default_rng(8100 + seed)
    for trial in range(6):
        n = int(rng.integers(1, 400))
        caps = rng.integers(0, (4, 9, 30)[trial % 3], size=n)
        cpu = (caps * 1000 + rng.integers(0, 1000, size=n)).astype(np.int64)
        mem = np.full(n, 1 << 40, np.int64)
        gpu = np.zeros(n, np.int64)
        if seed % 4 == 3:
            cpu[rng.integers(0, n)] = -5
        exec_idx = rng.permutation(n)[: max(1, int(n * rng.uniform(0.5, 1.0)))].astype(np.int32)
        drv_idx = rng.permutation(n)[: max(1, int(n * rng.uniform(0.2, 1.0)))].astype(np.int32)
        q = 200
        count = rng.integers(0, max(2, int(caps.sum()) + 3), size=q).astype(np.int32)
        count[::7] = rng.integers(0, 12, size=len(count[::7]))
        exe_cpu = np.full(q, 1000, np.int64)
        exe_mem = np.ones(q, np.int64)
        if seed % 4 == 2:
            exe_cpu[::3] = 0; exe_mem[::3] = 0
        apps = {"drv_cpu": rng.integers(0, 4000, size=q).astype(np.int64), "drv_mem": np.ones(q, np.int64),
                "drv_gpu": np.zeros(q, np.int64), "exe_cpu": exe_cpu, "exe_mem": exe_mem, "exe_gpu": np.zeros(q, np.int64),
                "count": count}
        packer.set_snapshot(cpu, mem, gpu, exec_idx, drv_idx)
        _, want, _ = _oracle_batch(oracle, MF_ORC, 0, cpu, mem, gpu, drv_idx, exec_idx, apps)
        got = packer.pack_batch(apps, MF_DEV, 0)
        assert_same_results(got, want, f"minfrag dense seed {seed} trial {trial}")


def test_minfrag_wide_capacities(oracle, packer):
    """general (64-bit) class: byte-granular requests against 2^40-scale nodes -> capacities far above 2^32, every division path"""
    rng = np.random.default_rng(8200)
    n = 96
    cpu = rng.integers(0, 1 << 40, n).astype(np.int64)
    mem = rng.integers(0, 1 << 45, n).astype(np.int64)
    gpu = np.zeros(n, np.int64)
    idx = np.arange(n, dtype=np.int32)
    exe_mem = np.array([1, 3, 1 << 20, (1 << 20) * 3, (1 << 33) + 1, (1 << 34) + 2, 7 << 31, 12345678901, 1 << 44, 5], np.int64)
    q = len(exe_mem) * 6
    apps = {"drv_cpu": np.full(q, 1000, np.int64), "drv_mem": np.full(q, 1 << 30, np.int64), "drv_gpu": np.zeros(q, np.int64),
            "exe_cpu": np.tile(np.array([1, 1000, 7, 0, 1 << 35, 3 << 33], np.int64), len(exe_mem)),
            "exe_mem": np.repeat(exe_mem, 6), "exe_gpu": np.zeros(q, np.int64),
            "count": rng.integers(1, 3000, q).astype(np.int32)}
    packer.set_snapshot(cpu, mem, gpu, idx, idx)
    _, want, _ = _oracle_batch(oracle, MF_ORC, 0, cpu, mem, gpu, idx, idx, apps)
    got = packer.pack_batch(apps, MF_DEV, 0)
    assert_same_results(got, want, "minfrag wide")


def test_minfrag_zones_as_groups_and_bench_shape(oracle, packer):
    """zones = instance groups (how single-az-minimal-fragmentation uses the entry) and the 10k-node bench shape"""
    import k8s_spark_scheduler_b200.synth as synth
    G = 4
    nodes = synth.make_nodes(900, groups=G)
    apps = synth.make_apps(600, groups=G)
    eoff, eorder = synth.group_orders(nodes)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "group")}
    dn, en, off = packer.pack_batch(a, MF_DEV, 0)
    for g in range(G):
        sel = np.nonzero(apps["group"] == g)[0]
        sub = {k: np.asarray(v)[sel] for k, v in a.items()}
        order = eorder[eoff[g]:eoff[g + 1]]
        _, (wd, we, woff), _ = _oracle_batch(oracle, MF_ORC, 0, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order, sub)
        assert np.array_equal(dn[sel], wd), g
        for j, i in enumerate(sel):
            if wd[j] >= 0:
                assert np.array_equal(en[off[i]:off[i + 1]], we[woff[j]:woff[j + 1]]), (g, i)
    nodes = synth.make_nodes(10000)
    apps = synth.make_apps(3000)
    order = synth.priority_order(nodes["avail_cpu"], nodes["avail_mem"])
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order)
    a = {k: apps[k] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count")}
    _, want, _ = _oracle_batch(oracle, MF_ORC, 0, nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], order, order, a)
    got = packer.pack_batch(a, MF_DEV, 0)
    assert_same_results(got, want, "minfrag bench shape")
    # same driver as tightly-pack: a driver candidate is feasible iff the capacities add up to k, for both packers
    tp = packer.pack_batch(a, 0, 0)
    assert np.array_equal(tp[0], got[0])


def test_minfrag_is_independent_mode_only(packer):
    from k8s_spark_scheduler_b200 import GangpackError
    idx = np.arange(2, dtype=np.int32)
    packer.set_snapshot([8000, 8000], [8 << 30, 8 << 30], [0, 0], idx, idx)
    base = {"drv_cpu": [1000], "drv_mem": [1 << 30], "drv_gpu": [0], "exe_cpu": [1000], "exe_mem": [1 << 30], "exe_gpu": [0], "count": [1]}
    for mode in (1, 2):
        with pytest.raises(GangpackError) as e:
            packer.pack_batch(base, MF_DEV, mode)
        assert e.value.status == 1
    dn, en, _ = packer.pack_batch(base, MF_DEV, 0)
    assert dn[0] == 0 and en[0] == 0


# ---------------------------------------------------------------------------------------------------------------
# executor reschedule (SURVEY §8f row f4): gp_reschedule_executors == rescheduleExecutor's node choice
# ---------------------------------------------------------------------------------------------------------------
def test_reschedule_goldens(golden, packer):
    for case in golden["resched_cases"]:
        names, cpu, mem, gpu = case_arrays(case["nodes"])
        order = order_indices(case["exec_order"], names)
        packer.set_snapshot(cpu, mem, gpu, order, order)
        idx = {n: i for i, n in enumerate(names)}
        reserved = None
        if case["overhead"]:
            reserved = [np.zeros(len(names), np.int64) for _ in range(3)]
            for k, v in case["overhead"].items():
                for d in range(3):
                    reserved[d][idx[k]] = v[d]
        exe = ([case["exe"][0]], [case["exe"][1]], [case["exe"][2]])
        got = packer.reschedule_executors(exe, min_frag=case["min_frag"], reserved=reserved,
                                          hosting=[[idx[h] for h in case["hosting"]]] if case["min_frag"] else None)
        want = idx[case["expect"]] if case["expect"] is not None else -1
        assert got[0] == want, case["id"]


@pytest.mark.parametrize("seed", range(4))
def test_reschedule_random(oracle, packer, seed):
    rng = np.random.default_rng(9100 + seed)
    for trial in range(6):
        n = int(rng.integers(1, 400))
        names = ["n%03d" % i for i in range(n)]
        cpu = (rng.integers(-1, 9, n) * 1000).astype(np.int64)
        mem = (rng.integers(0, 9, n) * (1 << 30) + rng.integers(0, 5, n)).astype(np.int64)
        gpu = rng.integers(0, 3, n).astype(np.int64)
        order = rng.permutation(n)[: int(rng.integers(1, n + 1))].astype(np.int32)
        packer.set_snapshot(cpu, mem, gpu, order, order)
        cl = oracle.Cluster(names, cpu, mem, gpu)
        onames = [names[i] for i in order]
        q = 64
        ec = (rng.integers(0, 4, q) * 1000).astype(np.int64)
        em = (rng.integers(0, 3, q) * (1 << 30) + (rng.integers(0, 3, q) == 0) * 3).astype(np.int64)
        eg = rng.integers(0, 2, q).astype(np.int64)
        res = [(rng.integers(0, 3, n) * 500).astype(np.int64), (rng.integers(0, 2, n) * (1 << 29)).astype(np.int64), np.zeros(n, np.int64)]
        over = {names[i]: (int(res[0][i]), int(res[1][i]), 0) for i in range(n)}
        hosting = [[int(x) for x in rng.permutation(n)[: int(rng.integers(0, 6))]] for _ in range(q)]
        ff = packer.reschedule_executors((ec, em, eg))
        mf = packer.reschedule_executors((ec, em, eg), min_frag=True, reserved=res, hosting=hosting)
        mf0 = packer.reschedule_executors((ec, em, eg), min_frag=True)
        for i in range(q):
            exe = (int(ec[i]), int(em[i]), int(eg[i]))
            w = cl.reschedule_executor(False, exe, onames)
            assert ff[i] == (names.index(w) if w else -1), (seed, trial, i, "first fit")
            w = cl.reschedule_executor(True, exe, onames, over, [names[h] for h in hosting[i]])
            assert mf[i] == (names.index(w) if w else -1), (seed, trial, i, "min frag")
            w = cl.reschedule_executor(True, exe, onames)
            assert mf0[i] == (names.index(w) if w else -1), (seed, trial, i, "min frag, no overhead / hosting")


def test_reschedule_groups_and_errors(oracle, packer):
    import k8s_spark_scheduler_b200.synth as synth
    from k8s_spark_scheduler_b200 import GangpackError
    G = 3
    nodes = synth.make_nodes(600, groups=G)
    eoff, eorder = synth.group_orders(nodes)
    packer.set_snapshot(nodes["avail_cpu"], nodes["avail_mem"], nodes["avail_gpu"], eorder, eorder, eoff, eoff)
    names = synth.node_names(600)
    rng = np.random.default_rng(5)
    q = 90
    grp = rng.integers(0, G, q).astype(np.int32)
    ec = (rng.integers(1, 9, q) * 500).astype(np.int64); em = (rng.integers(1, 9, q) << 29).astype(np.int64)
    ff = packer.reschedule_executors((ec, em, None)[:2] + (np.zeros(q, np.int64),), group=grp)
    mf = packer.reschedule_executors((ec, em, np.zeros(q, np.int64)), min_frag=True, group=grp)
    for g in range(G):
        order = eorder[eoff[g]:eoff[g + 1]]
        cl = oracle.Cluster([names[i] for i in order], nodes["avail_cpu"][order], nodes["avail_mem"][order], nodes["avail_gpu"][order])
        onames = [names[i] for i in order]
        for i in np.nonzero(grp == g)[0]:
            exe = (int(ec[i]), int(em[i]), 0)
            w = cl.reschedule_executor(False, exe, onames)
            assert ff[i] == (names.index(w) if w else -1), (g, i)
            w = cl.reschedule_executor(True, exe, onames)
            assert mf[i] == (names.index(w) if w else -1), (g, i)
    with pytest.raises(GangpackError) as e:
        packer.reschedule_executors(([-1], [1], [0]))
    assert e.value.status == 1
    with pytest.raises(GangpackError) as e:
        packer.reschedule_executors(([1], [1], [0]), group=[7])
    assert e.value.status == 1
    with pytest.raises(GangpackError) as e:
        packer.reschedule_executors(([1], [1], [0]), min_frag=True, hosting=[[100000]])
    assert e.value.status == 1
    assert len(packer.reschedule_executors(([], [], []))) == 0
