"""Shared helpers for the parity tests (oracle <-> CUDA path)."""
import numpy as np

ALGO_ID = {"tightly-pack": 0, "distribute-evenly": 1}
MODE_ID = {"independent": 0, "reference": 1, "exact": 2}


def case_arrays(nodes):
    names = [n["name"] for n in nodes]
    cpu = np.array([n["cpu"] for n in nodes], np.int64)
    mem = np.array([n["mem"] for n in nodes], np.int64)
    gpu = np.array([n["gpu"] for n in nodes], np.int64)
    return names, cpu, mem, gpu


def order_indices(order, names, drop_unknown=True):
    """Node names -> indices; names missing from the metadata are dropped (they can host nothing:
    binpack.go:68-69, pack_tightly.go:51-52) -- this is what the Go shim does when marshalling."""
    idx = {n: i for i, n in enumerate(names)}
    return np.array([idx[n] for n in order if n in idx], np.int32)


def res_aos(cpu, mem, gpu):
    return np.ascontiguousarray(np.stack([np.asarray(cpu, np.int64), np.asarray(mem, np.int64),
                                          np.asarray(gpu, np.int64)], axis=1))


def random_cluster(rng, n, tight=False, gpus=False, negative=False):
    """Small random cluster with awkward values (odd byte counts, zero dims, negatives)."""
    cpu = rng.integers(0, 16, n) * 500
    mem = rng.integers(0, 33, n) * (1 << 29) + (rng.integers(0, 3, n) == 0) * rng.integers(0, 1000, n)
    if tight:
        cpu = rng.integers(0, 6, n) * 500
        mem = rng.integers(0, 9, n) * (1 << 30)
    gpu = rng.integers(0, 3, n) if gpus else np.zeros(n, np.int64)
    if negative:
        neg = rng.integers(0, 8, n) == 0
        cpu = np.where(neg, -rng.integers(1, 3000, n), cpu)
        gneg = rng.integers(0, 10, n) == 0
        gpu = np.where(gneg, -1, gpu)
    return cpu.astype(np.int64), mem.astype(np.int64), gpu.astype(np.int64)


def random_apps(rng, q, gpus=False, zero_dims=False, big_counts=False):
    drv_cpu = rng.integers(0, 5, q) * 500
    drv_mem = rng.integers(0, 5, q) * (1 << 29)
    exe_cpu = rng.integers(1, 9, q) * 250
    exe_mem = rng.integers(1, 17, q) * (1 << 28) + (rng.integers(0, 4, q) == 0) * rng.integers(1, 999, q)
    if zero_dims:
        exe_cpu = np.where(rng.integers(0, 4, q) == 0, 0, exe_cpu)
        exe_mem = np.where(rng.integers(0, 4, q) == 0, 0, exe_mem)
    drv_gpu = (rng.integers(0, 4, q) == 0).astype(np.int64) if gpus else np.zeros(q, np.int64)
    exe_gpu = (rng.integers(0, 3, q) == 0).astype(np.int64) if gpus else np.zeros(q, np.int64)
    count = rng.integers(0, 12, q)
    if big_counts:
        count = np.where(rng.integers(0, 5, q) == 0, rng.integers(30, 200, q), count)
    return {
        "drv_cpu": drv_cpu.astype(np.int64), "drv_mem": drv_mem.astype(np.int64), "drv_gpu": drv_gpu,
        "exe_cpu": exe_cpu.astype(np.int64), "exe_mem": exe_mem.astype(np.int64), "exe_gpu": exe_gpu,
        "count": count.astype(np.int32),
    }


def assert_same_results(got, want, label=""):
    """(driver_node, executor_nodes, off) tuples: bit-exact on drivers and on the ExecutorNodes of
    every app that fits."""
    gd, ge, goff = got
    wd, we, woff = want
    assert np.array_equal(goff, woff), label + " offsets differ"
    bad = np.nonzero(np.asarray(gd) != np.asarray(wd))[0]
    assert bad.size == 0, f"{label} driver_node differs at apps {bad[:10]}: got {np.asarray(gd)[bad[:10]]} want {np.asarray(wd)[bad[:10]]}"
    fits = np.asarray(wd) >= 0
    # compare executor slices of fitting apps only (others are unspecified)
    mask = np.zeros(int(woff[-1]), bool)
    for i in np.nonzero(fits)[0]:
        mask[woff[i]:woff[i + 1]] = True
    ge = np.asarray(ge)[:len(mask)]
    we = np.asarray(we)[:len(mask)]
    diff = np.nonzero((ge != we) & mask)[0]
    if diff.size:
        app = int(np.searchsorted(woff, diff[0], side="right") - 1)
        raise AssertionError(f"{label} executor_nodes differ first at app {app}: got {ge[woff[app]:woff[app+1]]} "
                             f"want {we[woff[app]:woff[app+1]]}")


def node_names(n):
    return ["node-%06d" % i for i in range(n)]


def literal_batch(oracle, algo, cpu, mem, gpu, drv_idx, exec_idx, apps, n_threads=8):
    """Independent batch through the LITERAL restatement (string-keyed maps, loop for loop: oracle/gangpack_oracle.c,
    following pack_tightly.go:45-61 / distribute_evenly.go:49-70 / binpack.go:60-87) -> (driver_node, executor_nodes, off)
    in node-table indices."""
    names = node_names(len(cpu))
    cl = oracle.Cluster(names, cpu, mem, gpu)
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"])
    exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    dn, en, off = cl.binpack_batch(algo, drv, exe, apps["count"], [names[i] for i in drv_idx], [names[i] for i in exec_idx],
                                   with_efficiencies=False, n_threads=n_threads)
    return dn, en, off


def group_slices(dn, en, off, sel):
    """The results of the applications `sel` (queue order) as their own batch: (driver_node, executor_nodes, off)."""
    sel = np.asarray(sel, np.int64)
    cnt = (off[sel + 1] - off[sel]).astype(np.int64)
    sub_off = np.zeros(len(sel) + 1, np.int64)
    np.cumsum(cnt, out=sub_off[1:])
    idx = np.repeat(off[sel] - sub_off[:-1], cnt) + np.arange(int(sub_off[-1]), dtype=np.int64)
    return np.asarray(dn)[sel], np.asarray(en)[idx], sub_off


def fifo_vs_closed(oracle, algo, mode, cpu, mem, gpu, eorder, dorder, eoff, doff, apps, got, label=""):
    """fitEarlierDrivers per instance group through the closed form: every driver_node (incl. -1 / -2) and every
    ExecutorNodes slice of `got` must match, group by group (the groups are disjoint node sets, so the oracle runs them
    one after the other on the availability the previous one left).  Returns the final (cpu, mem, gpu)."""
    dn, en, off = got
    group = np.asarray(apps.get("group", np.zeros(len(apps["count"]), np.int32)))
    avail = (np.asarray(cpu, np.int64), np.asarray(mem, np.int64), np.asarray(gpu, np.int64))
    for g in range(len(eoff) - 1):
        sel = np.nonzero(group == g)[0]
        if sel.size == 0:
            continue
        sub = {k: np.asarray(apps[k])[sel] for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count", "young")}
        drv = res_aos(sub["drv_cpu"], sub["drv_mem"], sub["drv_gpu"])
        exe = res_aos(sub["exe_cpu"], sub["exe_mem"], sub["exe_gpu"])
        _, wd, we, woff, avail = oracle.closed_batch(algo, mode, avail[0], avail[1], avail[2], dorder[doff[g]:doff[g + 1]],
                                                     eorder[eoff[g]:eoff[g + 1]], drv, exe, sub["count"], sub["young"])
        assert_same_results(group_slices(dn, en, off, sel), (wd, we, woff), f"{label} group {g}")
    return avail


def literal_fifo(oracle, algo, mode, cpu, mem, gpu, drv_idx, exec_idx, apps, young):
    """fitEarlierDrivers through the literal restatement -> ((driver_node, executor_nodes, off), final (cpu, mem, gpu))."""
    names = node_names(len(cpu))
    cl = oracle.Cluster(names, cpu, mem, gpu)
    drv = res_aos(apps["drv_cpu"], apps["drv_mem"], apps["drv_gpu"])
    exe = res_aos(apps["exe_cpu"], apps["exe_mem"], apps["exe_gpu"])
    _, dn, en, off = cl.fifo(algo, mode, drv, exe, apps["count"], young, [names[i] for i in drv_idx], [names[i] for i in exec_idx])
    return (dn, en, off), cl.available()
