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

LabelTable keeps every node's labels as the device's resident label table (gp_label_table_*) holds them, from node-informer
events, and encodes affinities against its interners for gp_match_node_affinity_resident.
"""
from __future__ import annotations

import re

import numpy as np

from .resident import ResidentTable

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


_i32, _i64, _u8 = (lambda x: np.asarray(x, np.int32)), (lambda x: np.asarray(x, np.int64)), (lambda x: np.asarray(x, np.uint8))


def _node_index(node_names) -> dict:
    name_to_node = {nm: i for i, nm in enumerate(node_names)}
    if len(name_to_node) != len(node_names) or "" in name_to_node:
        raise ValueError("node names must be unique and non-empty")
    return name_to_node


def encode(nodes, affinities) -> dict:
    """-> the gp_node_labels and gp_node_affinities arrays (numpy) plus n_keys / n_values."""
    keys, vals = _Ids(), _Ids()
    name_to_node = _node_index([nd["name"] for nd in nodes])

    label_off, label_key, label_val, label_ok, label_int = [0], [], [], [], []
    for nd in nodes:
        ent = sorted((keys.id(k), vals.id(v), v) for k, v in nd.get("labels", {}).items())
        for k, v, s in ent:
            ok, iv = parse_int(s)
            label_key.append(k); label_val.append(v); label_ok.append(ok); label_int.append(iv if ok else 0)
        label_off.append(len(label_key))

    progs = _encode_programs(affinities, keys.id, vals.id, name_to_node)
    return dict(n_nodes=len(nodes), n_keys=len(keys), n_values=len(vals),
                label_off=_i64(label_off), label_key=_i32(label_key), label_val=_i32(label_val), label_int_ok=_u8(label_ok),
                label_int=_i64(label_int), **progs)


def _encode_programs(affinities, key_id, val_id, name_to_node) -> dict:
    """the gp_node_affinities arrays of the affinities, with label keys and values mapped to ids by key_id / val_id and
    metadata.name to a node index by name_to_node"""
    sel_off, sel_key, sel_val, has_req, term_off = [0], [], [], [], [0]
    term_req_off, term_err = [0], []
    req_op, req_key, req_int, req_val_off, req_val = [], [], [], [0], []

    def add_req(op, key=0, bound=0, values=()):
        req_op.append(op); req_key.append(key); req_int.append(bound)
        req_val.extend(sorted(set(values))); req_val_off.append(len(req_val))

    for aff in affinities:
        for k, v in (aff.get("nodeSelector") or {}).items():
            sel_key.append(key_id(k)); sel_val.append(val_id(v))
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
                    add_req(o, key_id(k), bound, [val_id(v) for v in vs] if o in (IN, NOT_IN) else ())
                for k, op, vs in fields:
                    if k == "metadata.name":
                        add_req(FIELD_NAME_IN if op == "In" else FIELD_NAME_NOT_IN, bound=name_to_node.get(vs[0], -1))
                    else:
                        # extractNodeFields sets metadata.name only: any other field reads "" -> a constant outcome
                        always = (vs[0] == "") == (op == "In")
                        add_req(FIELD_NAME_NOT_IN if always else FIELD_NAME_IN, bound=-1)
            term_req_off.append(len(req_op))
        term_off.append(len(term_err))

    return dict(n_aff=len(affinities), sel_off=_i64(sel_off), sel_key=_i32(sel_key), sel_val=_i32(sel_val),
                has_required=_u8(has_req), term_off=_i64(term_off), term_req_off=_i64(term_req_off), term_parse_error=_u8(term_err),
                req_op=_i32(req_op), req_key=_i32(req_key), req_int=_i64(req_int), req_val_off=_i64(req_val_off), req_val=_i32(req_val))


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

    # one pad entry: an absent key reads entry 0 under a false mask, which must exist even when no node has a label
    lval, lok, lint = (np.append(enc[k], 0) for k in ("label_val", "label_int_ok", "label_int"))
    lok = lok.astype(bool)
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


_UNKNOWN = 0                    # the key id and value id of a string no node carries: no row ever holds them


class LabelTable(ResidentTable):
    """Every node's labels as the resident label table keeps them, from the node informer's events: set_node(name, labels)
    for an add or an update (nothing changes when the labels are the same), delete_node(name).

    Key and value strings are interned for good (id 0 of each is reserved for strings no node carries, so encoding an
    affinity never changes the table); node names get ids that a deleted node hands to the next new one.  delta() -> the
    arrays of one gp_label_table_update: the rows of the nodes whose labels changed (a deleted node's row cleared) and the
    ParseInt columns of the values interned since the last delta; see ResidentTable."""

    name, writes = "label", ("row_node", "value_id")

    def __init__(self, n_node_ids=64, max_labels=16, n_keys=64, n_values=256):
        super().__init__(LabelMirror(), n_node_ids=n_node_ids, max_labels=max_labels, n_keys=n_keys, n_values=n_values)
        self.labels = {}                                # node name -> {key: value}, as the events gave them
        self._keys, self._vals = _Ids({None: _UNKNOWN}), _Ids({None: _UNKNOWN})
        self._parsed = [(False, 0)]                     # per value id: ParseInt of the string
        self._node = {}                                 # node name -> id
        self._row = []                                  # per id: ((key id, value id), ...) by key id
        self._free = []
        self._longest = 0                               # the most labels any row has held: a stride that fits every row
        self._dirty, self._new_vals = set(), []

    # ---- events
    def set_node(self, name, labels: dict):
        labels = dict(labels)
        if name in self.labels and self.labels[name] == labels:
            return
        self.labels[name] = labels
        at = self._node.get(name)
        if at is None:
            at = self._free.pop() if self._free else len(self._row)
            if at == len(self._row):
                self._row.append(())
            self._node[name] = at
        self._row[at] = tuple(sorted((self._key(k), self._val(v)) for k, v in labels.items()))
        self._longest = max(self._longest, len(self._row[at]))
        self._dirty.add(at)

    def delete_node(self, name):
        at = self._node.pop(name, None)
        if at is None:
            return
        del self.labels[name]
        self._row[at] = ()
        self._dirty.add(at)
        self._free.append(at)

    # ---- queries
    def node_ids(self, names) -> np.ndarray:
        """the table's ids of these node names; -1 for a node the table does not know (no labels)"""
        return np.array([self._node.get(n, -1) for n in names], np.int32)

    def encode_affinities(self, affinities, node_names) -> dict:
        """the gp_node_affinities arrays of the affinities against this table's ids: a key or value no node carries becomes
        the reserved id 0 (value sets deduplicated after that), metadata.name the index in node_names (the call's node table)"""
        key = lambda k: self._keys.get(k, _UNKNOWN)
        val = lambda v: self._vals.get(v, _UNKNOWN)
        return _encode_programs(affinities, key, val, _node_index(list(node_names)))

    def to_node_labels(self, node_ids) -> dict:
        return self.mirror.to_node_labels(node_ids)

    # ---- internals
    def _bounds(self):
        return dict(n_node_ids=len(self._row), max_labels=self._longest, n_keys=len(self._keys), n_values=len(self._vals))

    def _changes(self, replay):
        if replay:
            rows = [at for at, r in enumerate(self._row) if r]
            vals = list(range(1, len(self._vals)))
        else:
            rows, vals = sorted(self._dirty), self._new_vals
        off = np.zeros(len(rows) + 1, np.int64)
        np.cumsum([len(self._row[at]) for at in rows], out=off[1:])
        pairs = [kv for at in rows for kv in self._row[at]]
        d = {"row_node": _i32(rows), "row_off": off,
             "label_key": np.array([k for k, _ in pairs], np.int32), "label_val": np.array([v for _, v in pairs], np.int32),
             "value_id": _i32(vals), "value_int_ok": np.array([self._parsed[v][0] for v in vals], np.uint8),
             "value_int": np.array([self._parsed[v][1] for v in vals], np.int64)}
        self._dirty, self._new_vals = set(), []
        return d

    def _key(self, k):
        return self._keys.id(k)

    def _val(self, v):
        n = len(self._vals)
        at = self._vals.id(v)
        if at == n:
            ok, iv = parse_int(v)
            self._parsed.append((ok, iv if ok else 0))
            self._new_vals.append(at)
        return at


class LabelMirror:
    """What gp_label_table_update leaves on the device, with numpy: apply(delta) as the library would."""

    def __init__(self):
        self.size = None

    def apply(self, d: dict):
        if d.get("reset"):
            self.size = dict(d["reset"])
            z = self.size
            self.count = np.zeros(z["n_node_ids"], np.int32)
            self.key = np.zeros((z["n_node_ids"], z["max_labels"]), np.int32)
            self.val = np.zeros((z["n_node_ids"], z["max_labels"]), np.int32)
            self.val_int_ok = np.zeros(z["n_values"], np.uint8)
            self.val_int = np.zeros(z["n_values"], np.int64)
        off = d["row_off"]
        for i, r in enumerate(d["row_node"]):
            lo, hi = int(off[i]), int(off[i + 1])
            self.count[r] = hi - lo
            self.key[r, :hi - lo] = d["label_key"][lo:hi]
            self.val[r, :hi - lo] = d["label_val"][lo:hi]
        v = np.asarray(d["value_id"], np.int64)
        ok = np.asarray(d["value_int_ok"], np.uint8) != 0
        self.val_int_ok[v] = ok
        self.val_int[v] = np.where(ok, np.asarray(d["value_int"], np.int64), 0)

    def to_node_labels(self, node_ids) -> dict:
        """the per-call gp_node_labels arrays (encode()'s keys) equivalent to a resident call over node_ids: node i's labels
        are row node_ids[i] (none for -1), label_int_ok / label_int from the value columns"""
        ids = np.asarray(node_ids, np.int64)
        cnt = np.where(ids >= 0, self.count[np.maximum(ids, 0)], 0).astype(np.int64)
        off = np.zeros(len(ids) + 1, np.int64)
        np.cumsum(cnt, out=off[1:])
        rows = np.repeat(np.maximum(ids, 0), cnt)
        cols = np.arange(int(off[-1]), dtype=np.int64) - np.repeat(off[:-1], cnt)
        key, val = self.key[rows, cols], self.val[rows, cols]
        return dict(n_nodes=len(ids), n_keys=self.size["n_keys"], n_values=self.size["n_values"], label_off=off,
                    label_key=key.astype(np.int32), label_val=val.astype(np.int32), label_int_ok=self.val_int_ok[val].copy(),
                    label_int=self.val_int[val].copy())
