"""CPU checks of the overhead computer's model: the string restatement (tests/overhead_ref.py) against hand-derived vectors,
the product's event side (overhead.PodRecords), interning (overhead.encode) and numpy evaluator (overhead.evaluate) against
the restatement on random string clusters, and the ctypes mirrors of gp_node_overhead's structs against a C compiler."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import overhead_ref as ref
from k8s_spark_scheduler_b200 import overhead as oh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPARK = "spark-scheduler"


def pod(ns, name, node, cpu=0, mem=0, gpu=0, labels=None, sched="default-scheduler", init=(), uid=None):
    return {"uid": uid or f"{ns}/{name}", "namespace": ns, "name": name, "nodeName": node, "labels": labels or {},
            "schedulerName": sched, "containers": [{"cpu": cpu, "memory": mem, "nvidia.com/gpu": gpu}],
            "initContainers": [dict(zip(("cpu", "memory", "nvidia.com/gpu"), i)) for i in init]}


def app(a, role):
    return {"spark-app-id": a, "spark-role": role}


def both(pods, lister, rrs, soft, nodes, events=None):
    """-> the restatement's (overhead, nonsched, warned) and the product's, each side fed the same events"""
    comp, rec = ref.OverheadComputer(), oh.PodRecords()
    for kind, *args in (events or [("add", p) for p in pods]):
        getattr(comp, "on_" + kind)(*args)
        getattr(rec, kind)(*args)
    ov, ns, warned = comp.get_overhead_by_node(nodes, lister, rrs, soft)
    want = (ref.columns(nodes, ov), ref.columns(nodes, ns), warned)
    enc = oh.encode(rec.slots, lister, rrs, soft, nodes)
    g_ov, g_ns, has, g_warned = oh.evaluate(enc)
    got = (tuple(list(map(int, c)) for c in g_ov), tuple(list(map(int, c)) for c in g_ns), g_warned)
    return want, (tuple(got[0]), tuple(got[1]), got[2]), enc, has


def test_pod_to_resources_takes_the_init_container_max_per_dimension():
    p = pod("a", "p", "n", init=[(300, 5, 0), (100, 64, 2)])
    p["containers"] = [{"cpu": 100, "memory": 10}, {"cpu": 50, "memory": 20, "nvidia.com/gpu": 1, "ephemeral-storage": 7}]
    assert ref.pod_to_resources(p) == [300, 64, 2]
    assert oh.pod_to_resources(p) == (300, 64, 2)
    assert oh.pod_to_resources(pod("a", "q", "n", 5, 6, 0)) == (5, 6, 0)


def _hand_cluster():
    A = pod("a", "ds", "n1", 100, 10, init=[(300, 5, 0)])                               # (300, 10, 0), no labels
    B = pod("a", "app1-driver", "n1", 1000, 100, labels=app("app1", "driver"), sched=SPARK)  # in RR (a, app1)
    C = pod("a", "app1-exec-1", "n1", 2000, 200, labels=app("app1", "executor"), sched=SPARK)  # no reservation: warned
    D = pod("b", "x-exec", "n2", 500, 50, 1, labels=app("app1", "executor"), sched=SPARK)  # RR (a, app1) lists it: other ns
    E = pod("b", "y-exec", "n2", 600, 60, labels=app("app1", "executor"), sched=SPARK)     # soft["app1"]: across namespaces
    F = pod("a", "app1-drv2", "n2", 400, 40, labels=app("app1", "driver"), sched=SPARK)    # a driver named in the soft store
    G = pod("a", "gone", "n1", 70, 7)                                                       # absent from the lister
    H = pod("a", "ds3", "n3", 80, 8)                                                        # on a node not listed
    I = pod("a", "lonely", "n2", 7, 1, labels={"spark-role": "executor"}, sched=SPARK)     # no app label
    pods = [A, B, C, D, E, F, G, H, I]
    lister = {(p["namespace"], p["name"]): p for p in pods if p is not G}
    rrs = {("a", "app1"): ["app1-driver", "x-exec", "gone-exec"]}
    soft = {"app1": ["y-exec", "app1-drv2"]}
    return pods, lister, rrs, soft


def test_hand_derived_overhead():
    pods, lister, rrs, soft = _hand_cluster()
    nodes = ["n1", "n2"]
    want, got, enc, has = both(pods, lister, rrs, soft, nodes)
    expected = (([300 + 2000, 500 + 400 + 7], [10 + 200, 50 + 40 + 1], [0, 1]),   # overhead: A + C | D + F + I
                ([300, 0], [10, 0], [0, 0]),                                          # non-schedulable: A alone
                2)                                                                    # warned: C and F
    assert want == expected
    assert got == expected
    # has_reservation per slot: B (RR) and E (soft, across namespaces) only
    assert has.tolist() == [0, 1, 0, 0, 1, 0, 0, 0, 0]


def test_node_value_does_not_depend_on_the_other_listed_nodes():
    pods, lister, rrs, soft = _hand_cluster()
    _, alone, _, _ = both(pods, lister, rrs, soft, ["n2"])
    _, full, _, _ = both(pods, lister, rrs, soft, ["n3", "n1", "n2", "n4"])
    assert [c[0] for c in alone[0]] == [c[2] for c in full[0]]
    assert [c[1] for c in full[0]] == [300 + 2000, 210, 0] and [c[0] for c in full[0]] == [80, 8, 0]
    assert [c[3] for c in full[0]] == [0, 0, 0]                                          # a node without records


def test_bind_as_add_update_and_delete():
    unbound = pod("a", "late", "", 50, 5)
    bound = dict(unbound, nodeName="n1")
    resized = dict(bound, containers=[{"cpu": 999, "memory": 99}])
    lister = {("a", "late"): resized}
    steps = [("add", unbound), ("update", unbound, bound), ("update", bound, resized)]
    want, got, _, _ = both([], lister, {}, {}, ["n1"], events=steps)
    assert want == got == (([50], [5], [0]), ([50], [5], [0]), 0)               # the requests of the add event stay
    want, got, enc, _ = both([], lister, {}, {}, ["n1"], events=steps + [("delete", resized)])
    assert want == got == (([0], [0], [0]), ([0], [0], [0]), 0)
    assert enc["node_id"].tolist() == [-1]                                        # the slot is free
    want, got, _, _ = both([], lister, {}, {}, ["n1"], events=steps + [("update", resized, dict(resized, nodeName=""))])
    assert want == got == (([0], [0], [0]), ([0], [0], [0]), 0)                  # unbinding deletes


def test_free_slots_are_reused():
    rec = oh.PodRecords()
    p1, p2, p3 = pod("a", "p1", "n1", 1), pod("a", "p2", "n1", 2), pod("a", "p3", "n2", 3)
    for p in (p1, p2):
        rec.add(p)
    rec.delete(p1)
    rec.delete(pod("a", "p2", "n9", uid=p2["uid"]))     # another node's map: the reference finds nothing to delete
    rec.add(p3)
    assert [s and s[1] for s in rec.slots] == ["p3", "p2"]


def _random_cluster(rng, n_nodes, n_pods):
    nss, apps = ["ns0", "ns1", "ns2"], [f"app{i}" for i in range(6)]
    pods = []
    for k in range(n_pods):
        labels = {}
        if rng.random() < 0.8:
            labels["spark-app-id"] = apps[rng.integers(len(apps))]
        if rng.random() < 0.7:
            labels["spark-role"] = "executor" if rng.random() < 0.7 else "driver"
        init = [tuple(int(x) for x in rng.integers(0, 2000, 3))] if rng.random() < 0.3 else ()
        pods.append(pod(nss[rng.integers(3)], f"p{rng.integers(n_pods)}", f"n{rng.integers(n_nodes + 2)}",
                        int(rng.integers(0, 4000)), int(rng.integers(0, 1 << 34)), int(rng.integers(0, 3)), labels,
                        SPARK if rng.random() < 0.6 else "other", init, uid=f"u{k}"))
    lister = {}
    for p in pods:
        if rng.random() < 0.9:
            q = dict(p)
            if rng.random() < 0.1:                                   # the lister's current pod differs from the add event
                q["schedulerName"] = SPARK if p["schedulerName"] != SPARK else "other"
            lister[(p["namespace"], p["name"])] = q
    names = [p["name"] for p in pods] + ["zz"]
    rrs = {(nss[rng.integers(3)], a): list(rng.choice(names, int(rng.integers(0, 8)))) for a in apps if rng.random() < 0.7}
    soft = {a: list(rng.choice(names, int(rng.integers(0, 8)))) for a in apps if rng.random() < 0.6}
    events = []
    for p in pods:
        if rng.random() < 0.2:
            events += [("add", dict(p, nodeName="")), ("update", dict(p, nodeName=""), p)]
        else:
            events.append(("add", p))
        if rng.random() < 0.1:
            events.append(("delete", p))
    nodes = [f"n{i}" for i in rng.permutation(n_nodes)]
    return pods, lister, rrs, soft, nodes, events


@pytest.mark.parametrize("seed", range(40))
def test_encode_and_evaluate_match_the_restatement(seed):
    rng = np.random.default_rng(seed)
    pods, lister, rrs, soft, nodes, events = _random_cluster(rng, 1 + seed % 7, 5 + 7 * seed)
    want, got, _, _ = both(pods, lister, rrs, soft, nodes, events)
    assert want == got


def test_synthetic_cluster_matches_the_restatement():
    nodes, rec, lister, rrs, soft, pods = oh.synthetic_cluster(7, 200, 6000, big_apps=2, big_executors=300)
    comp = ref.OverheadComputer()
    for p in pods:
        comp.on_add(p)
    ov, ns, warned = comp.get_overhead_by_node(nodes, lister, rrs, soft)
    g_ov, g_ns, has, g_warned = oh.evaluate(oh.encode(rec.slots, lister, rrs, soft, nodes))
    assert [list(map(int, c)) for c in g_ov] == list(ref.columns(nodes, ov))
    assert [list(map(int, c)) for c in g_ns] == list(ref.columns(nodes, ns))
    assert g_warned == warned and warned > 0 and 0 < has.sum() < len(has)


def test_evaluate_refuses_a_sum_at_2_61():
    lister, pods = {}, [pod("a", f"p{i}", "n1", 1 << 60) for i in range(2)]
    for p in pods:
        lister[("a", p["name"])] = p
    rec = oh.PodRecords()
    for p in pods:
        rec.add(p)
    with pytest.raises(OverflowError):
        oh.evaluate(oh.encode(rec.slots, lister, {}, {}, ["n1"]))
    rec.slots[1] = ("a", "p1", "n1", ((1 << 60) - 1, 0, 0))
    assert int(oh.evaluate(oh.encode(rec.slots, lister, {}, {}, ["n1"]))[0][0][0]) == (1 << 61) - 1


def test_overhead_struct_layout_matches_header():
    from k8s_spark_scheduler_b200 import native
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gangpack.h"
    int main(void) {
      printf("%zu %zu %zu\n", sizeof(gp_overhead_pods), sizeof(gp_overhead_reservations), sizeof(gp_overhead_out));
      printf("%zu %zu %zu %zu %zu %zu\n", offsetof(gp_overhead_pods, node_id), offsetof(gp_overhead_pods, spark_scheduler),
             offsetof(gp_overhead_reservations, rr_app_key), offsetof(gp_overhead_reservations, soft_pod_name),
             offsetof(gp_overhead_out, has_reservation), offsetof(gp_overhead_out, n_warned));
      return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c, exe = os.path.join(td, "t.c"), os.path.join(td, "t")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        lines = subprocess.check_output([exe], text=True).split("\n")
    assert [int(x) for x in lines[0].split()] == [ctypes.sizeof(native.gp_overhead_pods), ctypes.sizeof(native.gp_overhead_reservations),
                                                  ctypes.sizeof(native.gp_overhead_out)]
    assert [int(x) for x in lines[1].split()] == [native.gp_overhead_pods.node_id.offset, native.gp_overhead_pods.spark_scheduler.offset,
                                                  native.gp_overhead_reservations.rr_app_key.offset,
                                                  native.gp_overhead_reservations.soft_pod_name.offset,
                                                  native.gp_overhead_out.has_reservation.offset, native.gp_overhead_out.n_warned.offset]
