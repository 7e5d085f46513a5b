"""Required node affinity without a GPU: the string oracle (tests/affinity_ref.py) against hand-derived vectors, and the
interning helper (affinity.encode) plus its numpy evaluator against the oracle on random string clusters."""
import numpy as np
import pytest

import affinity_ref as ar
import k8s_spark_scheduler_b200 as g
from k8s_spark_scheduler_b200 import affinity as aff

N0 = {"name": "n0", "labels": {"zone": "a", "ig": "batch", "gpus": "8", "odd": "x7"}}
N1 = {"name": "n1", "labels": {"zone": "b", "ig": "batch"}}
N2 = {"name": "n2", "labels": {}}


def term(*exprs, fields=()):
    return {"matchExpressions": list(exprs), "matchFields": list(fields)}


@pytest.mark.parametrize("s,want", [
    ("5", (5, False)), ("+5", (5, False)), ("007", (7, False)), ("-0", (0, False)), (" 5", (0, True)), ("5 ", (0, True)),
    ("", (0, True)), ("+", (0, True)), ("-", (0, True)), ("1_000", (0, True)), ("0x10", (0, True)), ("٣", (0, True)),
    ("9223372036854775807", (9223372036854775807, False)), ("9223372036854775808", (9223372036854775807, True)),
    ("-9223372036854775808", (-9223372036854775808, False)), ("-9223372036854775809", (-9223372036854775808, True)),
    ("99999999999999999999999", (0, True)),
])
def test_parse_int(s, want):
    assert ar.parse_int(s) == want
    assert aff.parse_int(s)[0] == (not want[1])
    if not want[1]:
        assert aff.parse_int(s)[1] == want[0]


def test_no_required_affinity_and_selector():
    assert ar.match({"nodeSelector": None, "required": None}, N2) == (True, False)
    assert ar.match({"nodeSelector": {"zone": "a"}, "required": None}, N0) == (True, False)
    assert ar.match({"nodeSelector": {"zone": "a"}, "required": None}, N1) == (False, False)
    assert ar.match({"nodeSelector": {"zone": "a"}, "required": None}, N2) == (False, False)


def test_empty_required_affinity_matches_no_node():
    # every term empty: all dropped at parse time, no term can match -> no match, and no error
    for terms in ([], [term()], [term(), {"matchExpressions": None, "matchFields": None}]):
        for node in (N0, N1, N2):
            assert ar.match({"required": terms}, node) == (False, False)


def test_not_in_on_absent_key_matches():
    p = {"required": [term(("gpus", "NotIn", ["8"]))]}
    assert ar.match(p, N2) == (True, False)
    assert ar.match(p, N1) == (True, False)
    assert ar.match(p, N0) == (False, False)


def test_selector_mismatch_masks_parse_error():
    p = {"nodeSelector": {"zone": "a"}, "required": [term(("zone", "Bogus", []))]}
    assert ar.match(p, N1) == (False, False)      # selector fails first: no error
    assert ar.match(p, N0) == (False, True)


def test_error_only_when_no_term_matched():
    bad = term(("zone", "In", []))                # In without values: NewRequirement error
    p = {"required": [bad, term(("zone", "In", ["a"]))]}
    assert ar.match(p, N0) == (True, False)       # a later term matched: the error is dropped
    assert ar.match(p, N1) == (False, True)
    assert ar.match({"required": [term(("zone", "In", ["a"])), bad]}, N0) == (True, False)


def test_gt_lt_on_non_integer_values():
    assert ar.match({"required": [term(("gpus", "Gt", ["4"]))]}, N0) == (True, False)
    assert ar.match({"required": [term(("gpus", "Lt", ["4"]))]}, N0) == (False, False)
    assert ar.match({"required": [term(("odd", "Gt", ["4"]))]}, N0) == (False, False)     # node value does not parse
    assert ar.match({"required": [term(("gpus", "Gt", ["4"]))]}, N2) == (False, False)    # key absent
    assert ar.match({"required": [term(("gpus", "Gt", ["x"]))]}, N0) == (False, True)     # bound does not parse: parse error
    assert ar.match({"required": [term(("gpus", "Gt", ["1", "2"]))]}, N0) == (False, True)
    # a bound must parse AND be a valid label value: a sign is not allowed there, so every negative bound is a parse error
    for bound, want in (("007", True), ("+7", None), ("-0", None), ("-1", None), (" 5", None), ("9223372036854775808", None)):
        got = ar.match({"required": [term(("gpus", "Gt", [bound]))]}, N0)
        assert got == ((True, False) if want else (False, True)), bound
    # node values: ParseInt's syntax alone ("+5", "-0" are not valid label values, but node labels are not validated here)
    for v, want in (("+5", True), ("007", True), ("-0", False), (" 5", False), ("9223372036854775808", False)):
        node = {"name": "v", "labels": {"gpus": v}}
        assert ar.match({"required": [term(("gpus", "Gt", ["4"]))]}, node) == (want, False), v
        assert ar.match({"required": [term(("gpus", "Lt", ["4"]))]}, node) == (v in ("-0",), False), v


def test_name_fields():
    p = {"required": [term(fields=[("metadata.name", "In", ["n1"])])]}
    assert [ar.match(p, n)[0] for n in (N0, N1, N2)] == [False, True, False]
    p = {"required": [term(fields=[("metadata.name", "NotIn", ["n1"])])]}
    assert [ar.match(p, n)[0] for n in (N0, N1, N2)] == [True, False, True]
    assert ar.match({"required": [term(fields=[("metadata.name", "In", ["n0", "n1"])])]}, N0) == (False, True)
    assert ar.match({"required": [term(fields=[("metadata.name", "Exists", [])])]}, N0) == (False, True)
    # other field keys read "" (only metadata.name is set)
    assert ar.match({"required": [term(fields=[("spec.x", "In", [""])])]}, N0) == (True, False)
    assert ar.match({"required": [term(fields=[("spec.x", "NotIn", ["v"])])]}, N0) == (True, False)
    assert ar.match({"required": [term(fields=[("spec.x", "In", ["v"])])]}, N0) == (False, False)
    # label and field requirements of one term must both hold
    p = {"required": [term(("ig", "In", ["batch"]), fields=[("metadata.name", "In", ["n1"])])]}
    assert [ar.match(p, n)[0] for n in (N0, N1, N2)] == [False, True, False]


def test_key_and_value_validation():
    assert not ar.is_qualified_name("example.com/MyName") and not ar.is_qualified_name("a")
    for bad in ("", "/a", "a/", "a/b/c", "-a", "a-", "Example.com/a", "a" * 64, "a\n"):
        assert ar.is_qualified_name(bad), bad
        assert not aff.valid_label_key(bad), bad
    for good in ("", "a", "a.b-c_d", "0" * 63):
        assert not ar.is_valid_label_value(good) and aff.valid_label_value(good)
    for bad in ("-a", "a b", "a" * 64, "a\n"):
        assert ar.is_valid_label_value(bad) and not aff.valid_label_value(bad)
    assert ar.match({"required": [term(("-bad", "Exists", []))]}, N0) == (False, True)
    assert ar.match({"required": [term(("zone", "Exists", ["a"]))]}, N0) == (False, True)
    assert ar.match({"required": [term(("zone", "In", ["bad value"]))]}, N0) == (False, True)


# ---- random string clusters: encode + numpy evaluator == oracle ----------------------------------------------------------
KEYS = ["zone", "ig", "gpus", "tier", "example.com/pool", "rank", "absent"]
VALUES = ["a", "b", "c", "batch", "web", "0", "7", "+5", "007", "-0", " 5", "9223372036854775808", "-12", "x"]
BAD_KEYS = ["-bad", "a/b/c"]


def random_cluster(rng, n, n_aff):
    nodes = []
    for i in range(n):
        ks = rng.choice(KEYS[:-1], int(rng.integers(0, len(KEYS))), replace=False)
        nodes.append({"name": f"node-{i}", "labels": {str(k): str(rng.choice(VALUES)) for k in ks}})
    names = [nd["name"] for nd in nodes] + ["ghost"]
    ops = ["In", "NotIn", "Exists", "DoesNotExist", "Gt", "Lt"]

    def expr():
        r = rng.random()
        key = str(rng.choice(BAD_KEYS)) if r < 0.03 else str(rng.choice(KEYS))
        op = str(rng.choice(ops + ["Bogus"] if rng.random() < 0.03 else ops))
        if op in ("In", "NotIn"):
            vals = [str(v) for v in rng.choice(VALUES, int(rng.integers(0 if rng.random() < 0.05 else 1, 4)), replace=False)]
        elif op in ("Gt", "Lt"):
            vals = [str(rng.choice(["3", "-1", "6", "x", "+2"]))]
        else:
            vals = [] if rng.random() > 0.05 else ["a"]
        return key, op, vals

    def field():
        op = "In" if rng.random() < 0.5 else ("NotIn" if rng.random() < 0.95 else "Exists")
        key = "metadata.name" if rng.random() < 0.85 else "spec.other"
        vals = [str(rng.choice(names + [""]))] if rng.random() > 0.05 else ["a", "b"]
        return key, op, vals

    affs = []
    for _ in range(n_aff):
        sel = {str(k): str(rng.choice(VALUES[:5])) for k in rng.choice(KEYS, int(rng.integers(0, 2)), replace=False)} \
            if rng.random() < 0.3 else None
        if rng.random() < 0.15:
            terms = None
        else:
            terms = [term(*[expr() for _ in range(int(rng.integers(0, 3)))],
                          fields=[field() for _ in range(int(rng.integers(0, 2)) if rng.random() < 0.3 else 0)])
                     for _ in range(int(rng.integers(0, 4)))]
        affs.append({"nodeSelector": sel, "required": terms})
    return nodes, affs


@pytest.mark.parametrize("seed", range(12))
def test_encoded_programs_equal_oracle(seed):
    rng = np.random.default_rng(seed)
    nodes, affs = random_cluster(rng, int(rng.integers(1, 90)), int(rng.integers(1, 40)))
    enc = aff.encode(nodes, affs)
    outcome, member, n_match, n_error = aff.evaluate(enc)
    want = np.array([[ar.outcome(p, nd) for nd in nodes] for p in affs], np.int8)
    assert np.array_equal(outcome, want)
    assert np.array_equal(aff.unpack_bits(member, len(nodes)), want == 1)
    assert np.array_equal(n_match, (want == 1).sum(1)) and np.array_equal(n_error, (want == 2).sum(1))
    # the encoding keeps the device's preconditions: keys ascending per node, value sets strictly ascending
    for i in range(len(nodes)):
        k = enc["label_key"][enc["label_off"][i]:enc["label_off"][i + 1]]
        assert np.all(np.diff(k) > 0)
    for r in range(len(enc["req_op"])):
        assert np.all(np.diff(enc["req_val"][enc["req_val_off"][r]:enc["req_val_off"][r + 1]]) > 0)


def test_outcome_kinds_all_occur():
    rng = np.random.default_rng(99)
    nodes, affs = random_cluster(rng, 60, 80)
    want = np.array([[ar.outcome(p, nd) for nd in nodes] for p in affs])
    assert {0, 1, 2} <= set(np.unique(want).tolist())


def test_pack_bits_roundtrip():
    rng = np.random.default_rng(3)
    for n in (1, 31, 32, 33, 100):
        m = rng.random((3, n)) < 0.5
        assert np.array_equal(aff.unpack_bits(aff.pack_bits(m), n), m)


def test_abi_declares_the_affinity_entries():
    assert {"gp_match_node_affinity", "gp_exceeds_cluster_capacity_affinity"} <= set(g.native.EXPORTS)
