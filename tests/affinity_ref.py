"""GetRequiredNodeAffinity(pod).Match(node), restated over strings: the checker of gp_match_node_affinity.

K8S = vendor/k8s.io.  match() follows RequiredNodeAffinity.Match (K8S/component-helpers/scheduling/corev1/nodeaffinity/
nodeaffinity.go:297-324), LazyErrorNodeSelector (:56-103), nodeSelectorTerm (:152-201), nodeSelectorRequirementsAsSelector /
AsFieldSelector (:203-280), labels.NewRequirement and Requirement.Matches (K8S/apimachinery/pkg/labels/selector.go:156-262),
fields.OneTerm(Not)EqualSelector, validation.IsQualifiedName / IsValidLabelValue, and strconv.ParseInt(s, 10, 64).

node = {"name": str, "labels": {str: str}}; pod = {"nodeSelector": {..} or None, "required": None or [term]},
term = {"matchExpressions": [(key, op, [values])], "matchFields": [(key, op, [values])]}.
-> (matched: bool, error: bool).
"""
from __future__ import annotations

import re

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def parse_int(s):
    """strconv.ParseInt(s, 10, 64): (value, err).  Sign '+' or '-', then ParseUint: base 10, so no '_' and no prefix."""
    if s == "":
        return 0, True
    neg = False
    if s[0] == "+":
        s = s[1:]
    elif s[0] == "-":
        neg, s = True, s[1:]
    if s == "":
        return 0, True
    n = 0
    for ch in s:
        if not ("0" <= ch <= "9"):
            return 0, True
        n = n * 10 + (ord(ch) - 48)
        if n > (1 << 64) - 1:
            return 0, True                             # ErrRange of ParseUint
    if not neg and n > INT64_MAX:
        return INT64_MAX, True
    if neg and n > -INT64_MIN:
        return INT64_MIN, True
    return (-n if neg else n), False


_QNAME_RE = re.compile(r"^([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]$")
_DNS1123_LABEL = r"[a-z0-9]([-a-z0-9]*[a-z0-9])?"
_DNS1123_SUBDOMAIN_RE = re.compile("^" + _DNS1123_LABEL + r"(\." + _DNS1123_LABEL + ")*$")
_LABEL_VALUE_RE = re.compile(r"^(([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9])?$")


def _full(rx, s):
    # Go's regexp '$' is end of text; Python's also matches before a final newline
    return "\n" not in s and rx.match(s) is not None


def is_qualified_name(value):
    errs = []
    parts = value.split("/")
    if len(parts) == 1:
        name = parts[0]
    elif len(parts) == 2:
        prefix, name = parts
        if len(prefix) == 0:
            errs.append("prefix empty")
        elif len(prefix) > 253 or not _full(_DNS1123_SUBDOMAIN_RE, prefix):
            errs.append("prefix not a subdomain")
    else:
        return ["too many slashes"]
    if len(name) == 0:
        errs.append("name empty")
    elif len(name) > 63:
        errs.append("name too long")
    if not _full(_QNAME_RE, name):
        errs.append("name format")
    return errs


def is_valid_label_value(value):
    errs = []
    if len(value) > 63:
        errs.append("too long")
    if not _full(_LABEL_VALUE_RE, value):
        errs.append("format")
    return errs


def new_requirement(key, op, vals):
    """labels.NewRequirement -> error?"""
    err = bool(is_qualified_name(key))
    if op in ("in", "notin"):
        err |= len(vals) == 0
    elif op in ("exists", "!"):
        err |= len(vals) != 0
    elif op in ("gt", "lt"):
        err |= len(vals) != 1
        err |= any(parse_int(v)[1] for v in vals)
    else:
        err = True
    err |= any(is_valid_label_value(v) for v in vals)
    return err


_OPS = {"In": "in", "NotIn": "notin", "Exists": "exists", "DoesNotExist": "!", "Gt": "gt", "Lt": "lt"}


def requirement_matches(key, op, vals, labels):
    """Requirement.Matches (selector.go:218-262)"""
    if op == "in":
        return key in labels and labels[key] in vals
    if op == "notin":
        return key not in labels or labels[key] not in vals
    if op == "exists":
        return key in labels
    if op == "!":
        return key not in labels
    if op in ("gt", "lt"):
        if key not in labels:
            return False
        lv, err = parse_int(labels[key])
        if err or len(vals) != 1:
            return False
        rv, err = parse_int(vals[0])
        if err:
            return False
        return lv > rv if op == "gt" else lv < rv
    return False


def parse_term(term):
    """newNodeSelectorTerm -> (label requirements or None, field requirements or None, parse error?)"""
    exprs, fields = term.get("matchExpressions") or [], term.get("matchFields") or []
    labels_sel, fields_sel, err = None, None, False
    if exprs:
        reqs, errs = [], False
        for key, op, vals in exprs:
            if op not in _OPS:
                errs = True
                continue
            if new_requirement(key, _OPS[op], vals):
                errs = True
            else:
                reqs.append((key, _OPS[op], list(vals)))
        if errs:
            err = True
        else:
            labels_sel = reqs
    if fields:
        sels, errs = [], False
        for key, op, vals in fields:
            if op in ("In", "NotIn") and len(vals) == 1:
                sels.append((key, op == "In", vals[0]))
            else:
                errs = True
        if errs:
            err = True
        else:
            fields_sel = sels
    return labels_sel, fields_sel, err


def match(pod, node):
    labels = node.get("labels", {})
    sel = pod.get("nodeSelector") or {}
    if len(sel) > 0:                                   # SelectorFromSet: one Equals requirement per entry
        for k, v in sel.items():
            if k not in labels or labels[k] != v:
                return False, False
    terms = pod.get("required")
    if terms is None:
        return True, False
    node_fields = {"metadata.name": node["name"]} if len(node["name"]) > 0 else {}
    errored = False
    for term in terms:
        if not (term.get("matchExpressions") or term.get("matchFields")):
            continue                                   # isEmptyNodeSelectorTerm: dropped at parse time
        lsel, fsel, err = parse_term(term)
        if err:
            errored = True
            continue
        if lsel is not None and not all(requirement_matches(k, op, vs, labels) for k, op, vs in lsel):
            continue
        if fsel is not None and len(node_fields) > 0 and not all(
                (node_fields.get(k, "") == v) == eq for k, eq, v in fsel):
            continue
        return True, False
    return False, errored


def outcome(pod, node):
    """0 no match, 1 match, 2 error"""
    m, e = match(pod, node)
    return 1 if m else (2 if e else 0)
