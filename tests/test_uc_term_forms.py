"""Register forms of the unique-condition evaluator (cb_specialize.h: generate_uc): size() and constant indices of list
attributes read from the list registers, ordering / equality / has() on register slots, startsWith / endsWith / contains
over two string attributes.  The generated text is compiled for the host (tests/hostsim) and must give oracle #2's bits
on requests whose attributes take every edge those forms branch on: list lengths around the 8 cached elements,
non-string elements, absent / string / map / number values, operands of 0 to 20 bytes from the table's and the batch's
string dictionaries."""
import random
import re

import numpy as np
import pytest

from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table.flatten import flatten
from hostsim import driver as hostsim
from oracle import cref

CONDITIONS = [
    "size(P.attr.l) == 0", "size(P.attr.l) == 1", "size(P.attr.l) >= 8", "size(P.attr.l) > 8", "size(P.attr.l) == 20",
    "size(P.attr.sz) > 2",                                   # read only through size(): a list slot of its own
    'P.attr.l[0] == "a"', 'P.attr.l[7] == "h"', 'P.attr.l[8] == "i"', "P.attr.l[0] in R.attr.m", "P.attr.l[7] in R.attr.m",
    "P.attr.s.startsWith(R.attr.p)", "P.attr.s.endsWith(R.attr.p)", "P.attr.s.contains(R.attr.p)",
    "has(R.attr.p)", "P.attr.n >= R.attr.k", "P.attr.n < R.attr.k", "R.attr.owner == P.id",
    'R.attr.p == "abcdefgh"',                                # an 8-byte string of the table dictionary
]
# operands: 0, 7, 8, 9 and 20 bytes, multi-byte UTF-8; some are table strings (the constants above), the rest batch strings
STRINGS = ["", "a", "abcdefg", "abcdefgh", "abcdefghi", "abcdefghijklmnopqrst", "bcdefgh", "ghi", "héllo✓", "✓", "h", "i",
           "xabcdefghijklmnopqrst", "abcdefghijklmnopqrstu", "qrst", "lmnopq"]
ELEMS = ["a", "b", "c", "d", "e", "f", "g", "h", "i", "j"]


def _value(r, kind):
    if kind == "absent":
        return None
    if kind == "str":
        return r.choice(STRINGS)
    if kind == "num":
        return r.choice([0, 1, 2.5, -3, 9])
    if kind == "map":
        return {"a": 1, "b": "x"}
    if kind == "bool":
        return r.random() < 0.5
    n = r.choice([0, 1, 2, 7, 8, 9, 20])
    base = [ELEMS[(j + r.randrange(3)) % len(ELEMS)] if r.random() < 0.8 else ELEMS[j % len(ELEMS)] for j in range(n)]
    if kind == "list_odd" and n:                              # a number / list / bool element somewhere
        base[r.randrange(n)] = r.choice([3, ["a"], True, 1.5])
    return base


def _request(r, i, n_actions):
    def pick(name, kinds):
        v = _value(r, r.choice(kinds))
        if v is not None:
            attrs[name] = v
    attrs = {}
    pick("l", ["list", "list", "list", "list_odd", "absent", "str", "map", "num"])
    pick("sz", ["list", "str", "map", "absent", "num", "list_odd"])
    pick("s", ["str", "str", "str", "num", "absent", "list"])
    pick("n", ["num", "num", "str", "absent"])
    p_attrs = attrs
    attrs = {}
    pick("m", ["list", "list", "list_odd", "absent", "str"])
    pick("p", ["str", "str", "str", "num", "absent", "bool"])
    pick("k", ["num", "num", "str", "absent"])
    if r.random() < 0.5:
        attrs["owner"] = f"p{i % 5}"
    return {"requestId": str(i), "actions": [f"a{j}" for j in range(n_actions)],
            "principal": {"id": f"p{r.randrange(5)}", "roles": ["user"], "attr": p_attrs},
            "resource": {"kind": "doc", "id": f"r{i}", "attr": attrs}}


def _table(negated=False):
    """One rule per condition; negated: every condition under `!`, so that a term's error and its false give different
    decisions (an error drops the whole condition, ruletable.go:1467-1486, a false under `!` satisfies it)."""
    conds = [f"!({e})" for e in CONDITIONS] if negated else CONDITIONS
    rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}} for i, e in enumerate(conds)]
    pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "doc", "version": "default", "rules": rules}}
    return flatten(build_rule_table([pol]))


def _edge_requests(table_last, start, n_actions):
    """startsWith / endsWith / contains operands at the ends of both dictionaries: the table's last string, and a fresh
    pair of strings in the last request, whose resource attribute `p` is the batch dictionary's last string."""
    def req(i, s, p):
        return {"requestId": str(i), "actions": [f"a{j}" for j in range(n_actions)],
                "principal": {"id": "p0", "roles": ["user"], "attr": {"s": s, "l": ["a"], "sz": ["a"], "n": 1}},
                "resource": {"kind": "doc", "id": "r0", "attr": {"p": p, "m": ["a"], "k": 1}}}
    pairs = [(table_last, table_last), (table_last + "x", table_last), ("x" + table_last, table_last), (table_last, table_last[:-1]),
             (table_last, table_last[1:]), (table_last[:-1], table_last), ("x", table_last), (table_last, "")]
    out = [req(start + j, s, p) for j, (s, p) in enumerate(pairs)]
    last_p = "zz-batch-dictionary-last"
    out += [req(start + len(out), "zz-batch-dictionary-last-but-one" + last_p, last_p)]
    return out


def _batch_strings(b):
    off = np.frombuffer(np.ascontiguousarray(b.columns[5]).tobytes(), dtype=np.uint32)
    raw = np.ascontiguousarray(b.columns[6]).tobytes()
    return [raw[off[j]:off[j + 1]].decode() for j in range(len(off) - 1)]


def _operator_body(src):
    return src[src.index("CB_HD CondWord operator()"):]


def test_forms_are_generated():
    ft = _table()
    src, nu = hostsim.generate_uc(ft.blob)
    assert nu == len(CONDITIONS) and src
    body = _operator_body(src)
    assert "term_operand(" not in body and body.count("term_tri(") == 1   # l[8]
    assert body.count("list_size(") == 6 and "str_tri(t, b, 2u" in body and "str_tri(t, b, 3u" in body and "str_tri(t, b, 4u" in body
    assert "has_tri(" in body and "ord_tri(" in body and "cmp_tri(" in body and "eq_tri(" in body
    # constant indices below the 8 cached elements come from the registers, l[8] takes the generic path
    assert len(re.findall(r"list_elem\(t, b, cols\.slot\(\d+u\), cols\.l\d+, [07]u\)", body)) == 4
    assert "uc_term_operand(" not in body and body.count("uc_term_tri(") == 1


def test_c3_terms_all_take_register_forms():
    import workloads as W
    _, ft, _ = W.build(W.C3())
    body = _operator_body(hostsim.generate_uc(ft.blob)[0])
    assert "term_tri(" not in body and "term_operand(" not in body


@pytest.mark.parametrize("negated", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_forms_against_oracle(seed, negated, tmp_path):
    ft = _table(negated)
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    r = random.Random(4400 + seed)
    enc = Encoder(ft.manifest)
    reqs = [_request(r, i, len(CONDITIONS)) for i in range(400)]
    reqs += _edge_requests(ft.manifest["strings"][-1], len(reqs), len(CONDITIONS))
    b = enc.encode(reqs)
    assert _batch_strings(b)[-1] == reqs[-1]["resource"]["attr"]["p"]
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for mode in (4, 5):
        got = hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode)
        assert (got == want).all(), (seed, negated, mode)
