"""Interning of node labels and required node affinities into the arrays of gp_match_node_affinity (include/gangpack.h).

This is what a caller does before the device sees anything: label keys and values become dense ids, and every rule that needs
the strings is applied here -- NewRequirement's validation (vendor/k8s.io/apimachinery/pkg/labels/selector.go:156-196) becomes
a term's parse_error flag, strconv.ParseInt of a node's label value becomes label_int_ok / label_int, and metadata.name becomes
a node index.

Description accepted by encode():
    nodes       [{"name": str, "labels": {key: value}}]                       (names unique and non-empty)
    affinities  [{"nodeSelector": {key: value} or None,
                  "required": None (no requiredDuringScheduling...) or [term, ...]}]
                term = {"matchExpressions": [(key, op, [values])], "matchFields": [(key, op, [values])]}

evaluate() runs the encoded programs with numpy on the host: the reference semantics over ids, used as a check of the device
and as the host baseline of tools/affinity_bench.py.
"""
from __future__ import annotations

import re

import numpy as np

IN, NOT_IN, EXISTS, DOES_NOT_EXIST, GT, LT, FIELD_NAME_IN, FIELD_NAME_NOT_IN = range(8)
_LABEL_OPS = {"In": IN, "NotIn": NOT_IN, "Exists": EXISTS, "DoesNotExist": DOES_NOT_EXIST, "Gt": GT, "Lt": LT}

_QNAME = re.compile(r"([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]")
_DNS1123_SUB = re.compile(r"[a-z0-9]([-a-z0-9]*[a-z0-9])?(\.[a-z0-9]([-a-z0-9]*[a-z0-9])?)*")
_INT64_MAX = (1 << 63) - 1


def parse_int(s: str):
    """strconv.ParseInt(s, 10, 64) -> (ok, value): an optional sign, then one or more ASCII digits, within int64."""
    body = s[1:] if s[:1] in ("+", "-") else s
    if not body or any(ch < "0" or ch > "9" for ch in body):
        return False, 0
    v = -int(body) if s[0] == "-" else int(body)
    return (-_INT64_MAX - 1 <= v <= _INT64_MAX), v


def valid_label_key(k: str) -> bool:
    """validation.IsQualifiedName: [DNS-1123 subdomain '/'] name, name <= 63 characters"""
    parts = k.split("/")
    if len(parts) > 2:
        return False
    name = parts[-1]
    if len(parts) == 2:
        prefix = parts[0]
        if not prefix or len(prefix) > 253 or not _DNS1123_SUB.fullmatch(prefix):
            return False
    return 0 < len(name) <= 63 and _QNAME.fullmatch(name) is not None


def valid_label_value(v: str) -> bool:
    """validation.IsValidLabelValue: empty, or a qualified-name part, <= 63 characters"""
    return len(v) <= 63 and (v == "" or _QNAME.fullmatch(v) is not None)


def _label_requirement_ok(key, op, values) -> bool:
    if op not in _LABEL_OPS or not valid_label_key(key):
        return False
    if op in ("In", "NotIn") and len(values) == 0:
        return False
    if op in ("Exists", "DoesNotExist") and len(values) != 0:
        return False
    if op in ("Gt", "Lt") and (len(values) != 1 or not all(parse_int(v)[0] for v in values)):
        return False
    return all(valid_label_value(v) for v in values)


class _Ids(dict):
    def id(self, s):
        return self.setdefault(s, len(self))


def encode(nodes, affinities) -> dict:
    """-> the gp_node_labels and gp_node_affinities arrays (numpy) plus n_keys / n_values."""
    keys, vals = _Ids(), _Ids()
    name_to_node = {nd["name"]: i for i, nd in enumerate(nodes)}
    if len(name_to_node) != len(nodes) or "" in name_to_node:
        raise ValueError("node names must be unique and non-empty")

    label_off, label_key, label_val, label_ok, label_int = [0], [], [], [], []
    for nd in nodes:
        ent = sorted((keys.id(k), vals.id(v), v) for k, v in nd.get("labels", {}).items())
        for k, v, s in ent:
            ok, iv = parse_int(s)
            label_key.append(k); label_val.append(v); label_ok.append(ok); label_int.append(iv if ok else 0)
        label_off.append(len(label_key))

    sel_off, sel_key, sel_val, has_req, term_off = [0], [], [], [], [0]
    term_req_off, term_err = [0], []
    req_op, req_key, req_int, req_val_off, req_val = [], [], [], [0], []

    def add_req(op, key=0, bound=0, values=()):
        req_op.append(op); req_key.append(key); req_int.append(bound)
        req_val.extend(sorted(set(values))); req_val_off.append(len(req_val))

    for aff in affinities:
        for k, v in (aff.get("nodeSelector") or {}).items():
            sel_key.append(keys.id(k)); sel_val.append(vals.id(v))
        sel_off.append(len(sel_key))
        terms = aff.get("required")
        has_req.append(terms is not None)
        for term in terms or []:
            exprs, fields = term.get("matchExpressions") or [], term.get("matchFields") or []
            bad = not all(_label_requirement_ok(k, op, vs) for k, op, vs in exprs)
            bad = bad or not all(op in ("In", "NotIn") and len(vs) == 1 for _, op, vs in fields)
            term_err.append(bad)
            if not bad:
                for k, op, vs in exprs:
                    o = _LABEL_OPS[op]
                    bound = parse_int(vs[0])[1] if o in (GT, LT) else 0
                    add_req(o, keys.id(k), bound, [vals.id(v) for v in vs] if o in (IN, NOT_IN) else ())
                for k, op, vs in fields:
                    if k == "metadata.name":
                        add_req(FIELD_NAME_IN if op == "In" else FIELD_NAME_NOT_IN, bound=name_to_node.get(vs[0], -1))
                    else:
                        # extractNodeFields sets metadata.name only: any other field reads "" -> a constant outcome
                        always = (vs[0] == "") == (op == "In")
                        add_req(FIELD_NAME_NOT_IN if always else FIELD_NAME_IN, bound=-1)
            term_req_off.append(len(req_op))
        term_off.append(len(term_err))

    i32, i64, u8 = (lambda x: np.asarray(x, np.int32)), (lambda x: np.asarray(x, np.int64)), (lambda x: np.asarray(x, np.uint8))
    return dict(n_nodes=len(nodes), n_keys=len(keys), n_values=len(vals), n_aff=len(affinities),
                label_off=i64(label_off), label_key=i32(label_key), label_val=i32(label_val), label_int_ok=u8(label_ok),
                label_int=i64(label_int), sel_off=i64(sel_off), sel_key=i32(sel_key), sel_val=i32(sel_val),
                has_required=u8(has_req), term_off=i64(term_off), term_req_off=i64(term_req_off), term_parse_error=u8(term_err),
                req_op=i32(req_op), req_key=i32(req_key), req_int=i64(req_int), req_val_off=i64(req_val_off), req_val=i32(req_val))


def evaluate(enc: dict):
    """numpy evaluation of the encoded programs -> (outcome[n_aff][n] in {0 no match, 1 match, 2 error}, member bitmap
    uint32[n_aff][words], n_match, n_error)."""
    n, A = enc["n_nodes"], enc["n_aff"]
    off = enc["label_off"]
    node_of = np.repeat(np.arange(n), np.diff(off))
    cache = {}

    def column(k):                      # per node: the label's entry index for key k, -1 = absent
        if k not in cache:
            col = np.full(n, -1, np.int64)
            hit = np.nonzero(enc["label_key"] == k)[0]
            col[node_of[hit]] = hit
            cache[k] = col
        return cache[k]

    lval, lok, lint = enc["label_val"], enc["label_int_ok"].astype(bool), enc["label_int"]
    idx = np.arange(n)
    outcome = np.zeros((A, n), np.int8)
    for a in range(A):
        ok = np.ones(n, bool)
        for t in range(enc["sel_off"][a], enc["sel_off"][a + 1]):
            e = column(int(enc["sel_key"][t]))
            ok &= (e >= 0) & (lval[np.maximum(e, 0)] == enc["sel_val"][t])
        if not enc["has_required"][a]:
            outcome[a] = ok
            continue
        matched, errored = np.zeros(n, bool), False
        for t in range(enc["term_off"][a], enc["term_off"][a + 1]):
            if enc["term_parse_error"][t]:
                errored = True
                continue
            r0, r1 = enc["term_req_off"][t], enc["term_req_off"][t + 1]
            if r0 == r1:
                continue
            tm = np.ones(n, bool)
            for r in range(r0, r1):
                op, bound = int(enc["req_op"][r]), int(enc["req_int"][r])
                if op == FIELD_NAME_IN:
                    tm &= idx == bound
                    continue
                if op == FIELD_NAME_NOT_IN:
                    tm &= idx != bound
                    continue
                e = column(int(enc["req_key"][r]))
                has = e >= 0
                es = np.maximum(e, 0)
                if op in (IN, NOT_IN):
                    inset = np.isin(lval[es], enc["req_val"][enc["req_val_off"][r]:enc["req_val_off"][r + 1]]) & has
                    tm &= inset if op == IN else ~inset
                elif op == EXISTS:
                    tm &= has
                elif op == DOES_NOT_EXIST:
                    tm &= ~has
                else:
                    good = has & lok[es]
                    tm &= good & ((lint[es] > bound) if op == GT else (lint[es] < bound))
            matched |= tm
        outcome[a] = np.where(~ok, 0, np.where(matched, 1, 2 if errored else 0))
    return outcome, pack_bits(outcome == 1), (outcome == 1).sum(1).astype(np.int32), (outcome == 2).sum(1).astype(np.int32)


def pack_bits(mask) -> np.ndarray:
    """bool[rows][n] -> uint32[rows][ceil(n / 32)], bit j % 32 of word j / 32"""
    mask = np.asarray(mask, bool)
    rows, n = mask.shape
    words = (n + 31) // 32
    padded = np.zeros((rows, words * 32), bool)
    padded[:, :n] = mask
    return np.packbits(padded.reshape(rows, words, 32), axis=-1, bitorder="little").view("<u4").reshape(rows, words).astype(np.uint32)


def unpack_bits(member, n) -> np.ndarray:
    """uint32[rows][words] -> bool[rows][n]"""
    m = np.asarray(member, np.uint32)
    return ((m[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(m.shape[0], -1)[:, :n]
