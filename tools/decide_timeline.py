#!/usr/bin/env python
"""Phase timeline of gp_decide_tables in one bench.py step: when the classify tiles, table items and decide chunks ran, how
long the phase waits took to notice their producers, and how long the decide tail is.  (diagnostic, not part of the bench
contract)

    python tools/decide_timeline.py [--workload tightly-100k] [--steps 20] [--root TREE] [--lib PATH [--prebuilt]]

It compiles the package's sources with -DGP_DECIDE_TIMELINE into a separate library (a temporary directory, or --lib;
never the in-tree libgangpack.so), runs the bench.py workload of --root (this checkout by default) through it, and reads
the %globaltimer stamps every CTA and warp wrote during the step's gp_decide_tables launch.  The instrumented build adds
a few stores per item and per warp; its step time is not the shipped build's.

Prints one JSON line: the GPU's name, power limit and maximum SM clock, and per metric the median over the steps with its
range.  Times are µs from the first ticket claim of the launch:
    cls / tab / decide          first start and last finish of the phase (tab: segments and first-fit items);
    cls_wait / tab_wait         spread of the CTAs' wait returns, and `gap`: first return after the phase's last item was
                                counted done (negative: the wait returned within one timer tick of it);
    decide_tail                 last warp's end minus the median warp's end;
    tickets                     ticket claims of the launch (items + one final claim per CTA)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

KINDS = {0: "cls", 1: "seg", 2: "firstfit", 3: "cls_wait", 4: "tab_wait"}
TL_CTAS, TL_PER_CTA, WARPS_PER_CTA = 1024, 48, 8     # gangpack_tables.cuh: kTlCtas, kTlPerCta, kTabThreads / 32


def tl_dtype():
    rec = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("kind", "<u4"), ("item", "<u4"), ("pad", "<u4", 2)])
    nw = TL_CTAS * WARPS_PER_CTA
    return np.dtype([("grid", "<u4"), ("n_cls", "<u4"), ("n_tab", "<u4"), ("n_chunks", "<u4"), ("n", "<u4", TL_CTAS),
                     ("rec", rec, (TL_CTAS, TL_PER_CTA)), ("warp", "<u8", (nw, 2)), ("warp_chunks", "<u4", nw)], align=True)


def step_metrics(buf):
    """One launch's timeline -> dict of metrics (µs from the first ticket claim)."""
    grid = int(buf["grid"])
    n = np.minimum(buf["n"][:grid], TL_PER_CTA)
    recs = np.concatenate([buf["rec"][b, :n[b]] for b in range(grid)])
    overflow = int((buf["n"][:grid] > TL_PER_CTA).sum())
    warp = buf["warp"][:grid * WARPS_PER_CTA]
    chunks = buf["warp_chunks"][:grid * WARPS_PER_CTA]
    busy = chunks > 0
    items = recs[recs["kind"] <= 2]
    t0 = int(items["t0"].min())
    us = lambda t: (np.asarray(t, np.float64) - t0) / 1e3
    m = {"grid": grid, "n_cls": int(buf["n_cls"]), "n_tab": int(buf["n_tab"]), "n_chunks": int(buf["n_chunks"]),
         "tickets": int(len(items) + grid), "records_dropped_ctas": overflow}
    cls = items[items["kind"] == 0]
    tab = items[items["kind"] >= 1]
    m["cls_first_start"], m["cls_last_done"] = float(us(cls["t0"].min())), float(us(cls["t1"].max()))
    if len(tab):
        m["tab_first_start"], m["tab_last_done"] = float(us(tab["t0"].min())), float(us(tab["t1"].max()))
    for kind, name, last in ((3, "cls_wait", m["cls_last_done"]), (4, "tab_wait", m.get("tab_last_done", m["cls_last_done"]))):
        w = recs[recs["kind"] == kind]
        if len(w):
            ret = us(w["t1"])
            m[name + "_first_return"], m[name + "_last_return"] = float(ret.min()), float(ret.max())
            m[name + "_spread"] = float(ret.max() - ret.min())
            m[name + "_gap"] = float(ret.min() - last)
            m[name + "_median_gap"] = float(np.median(ret) - last)
    if busy.any():
        s, e = us(warp[busy, 0]), us(warp[busy, 1])
        m["decide_first_start"], m["decide_last_end"] = float(s.min()), float(e.max())
        m["decide_median_end"] = float(np.median(e))
        m["decide_tail"] = float(e.max() - np.median(e))
        m["decide_warps"] = int(busy.sum())
        m["chunks_per_warp_max"] = int(chunks.max())
    stamps = np.unique(np.concatenate([recs["t0"], recs["t1"], warp[busy].ravel()]).astype(np.int64))
    d = np.diff(stamps)
    m["timer_step_ns"] = int(d[d > 0].min()) if (d > 0).any() else 0
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="tightly-100k")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--lib", default=None, help="where the instrumented library goes (default: a temporary directory)")
    ap.add_argument("--prebuilt", action="store_true", help="use --lib as it is (built earlier by this tool)")
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    tmp = None
    if args.lib is None:
        tmp = tempfile.TemporaryDirectory(prefix="gp_timeline_")
        args.lib = os.path.join(tmp.name, "libgangpack_timeline.so")
    lib = os.path.abspath(args.lib)
    # the package of `root` binds GANGPACK_LIB when it is imported
    os.environ["GANGPACK_LIB"] = lib
    sys.path.insert(0, root)
    import k8s_spark_scheduler_b200 as g
    if os.path.realpath(lib) == os.path.realpath(os.path.join(root, "k8s-spark-scheduler_b200", "libgangpack.so")):
        raise SystemExit("--lib must not be the in-tree libgangpack.so")
    if not args.prebuilt:
        g.native.build(force=True, out=lib, defines=("GP_DECIDE_TIMELINE",))
    if args.build_only:
        print(json.dumps({"built": lib}))
        return
    import torch
    from bench import WORKLOADS, make_workload

    L = g.native.load()
    L.gp_decide_timeline.restype = C.c_int64
    L.gp_decide_timeline.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    dt = tl_dtype()

    w = WORKLOADS[args.workload]
    nodes, a, eoff, eorder = make_workload(w, 0)
    dev = torch.device("cuda", 0)
    packer = g.GangPacker(device=0, async_snapshot=True)
    if L.gp_decide_timeline(packer._h, None, 0) != dt.itemsize:
        raise SystemExit("timeline layout of the library and of this tool differ")
    stream = torch.cuda.ExternalStream(packer.stream_handle(), device=dev)

    def t(x, dtype):
        return torch.from_numpy(np.ascontiguousarray(x)).to(dtype).to(dev)

    tn = {"cpu": t(nodes["avail_cpu"], torch.int64), "mem": t(nodes["avail_mem"], torch.int64), "gpu": t(nodes["avail_gpu"], torch.int64),
          "eorder": t(eorder, torch.int32), "eoff": t(eoff, torch.int32)}
    keys = ["drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu", "count"] + (["group"] if w["groups"] > 1 else [])
    ta = {k: t(a[k], torch.int64 if a[k].dtype == np.int64 else torch.int32) for k in keys}
    ta["off"] = t(a["off"], torch.int64)
    q = len(a["count"])
    d_driver = torch.empty(q, dtype=torch.int32, device=dev)
    d_exec = torch.empty(max(int(a["off"][-1]), 1), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()

    def step():
        packer.set_snapshot_device(tn["cpu"], tn["mem"], tn["gpu"], tn["eoff"], tn["eorder"], tn["eoff"], tn["eorder"])
        packer.pack_batch_device(ta, w["algo"], w["mode"], d_driver, d_exec)

    buf = np.zeros(1, dt)
    per = []
    with torch.cuda.stream(stream):
        for _ in range(10):
            step()
        torch.cuda.synchronize()
        for _ in range(args.steps):
            step()
            if L.gp_decide_timeline(packer._h, buf.ctypes.data, dt.itemsize) != dt.itemsize:
                raise SystemExit("gp_decide_timeline failed")
            per.append(step_metrics(buf[0]))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    summary = {}
    for k in per[0]:
        v = np.array([p[k] for p in per if k in p], np.float64)
        summary[k] = {"median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}
    print(json.dumps({"root": root, "workload": args.workload, "gpu": smi, "steps": args.steps, "timeline_us": summary}))
    torch.cuda.synchronize()
    packer.close()


if __name__ == "__main__":
    main()
