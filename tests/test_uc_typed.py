"""The typed branch of the unique-condition evaluator (cb_specialize.h: generate_uc): when every slot the flat terms read
has one type, load() keeps typed payloads and a per-request guard, and the terms are plain booleans under it; a request
that fails the guard evaluates the tri-state terms.  C3 takes the branch for all twelve slots; its requests are checked
against oracle #2 as they come (every lane typed) and with slots perturbed to every edge of the guard, typed and
perturbed lanes mixed inside each warp, on the host build and on the device."""
import math
import os
import random
import re

import numpy as np
import pytest

from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table.flatten import flatten
from hostsim import driver as hostsim
from oracle import cref

C3_TYPES = {"typed_str": [0, 1, 6, 7, 8, 10, 11], "typed_num": [4, 5], "typed_bool": [9]}
C3_LISTS = {2: 1, 3: 0}   # list slot -> elements its constant indices need (P.attr.groups[0])


def _c3():
    import workloads as W
    w = W.C3()
    _, ft, _ = W.build(w)
    return w, ft


def test_c3_takes_the_typed_branch_for_every_slot():
    _, ft = _c3()
    src = hostsim.generate_uc(ft.blob)[0]
    guard = re.search(r"r\.typed = (.*);", src).group(1).split(" & ")
    assert len(guard) == 12
    for fn, slots in C3_TYPES.items():
        for v in slots:
            assert f"{fn}(r.s{v})" in guard, (fn, v)
    for v, need in C3_LISTS.items():
        assert f"typed_list(r.l{v}, {need}u)" in guard
    body = src[src.index("CB_HD CondWord operator()"):]
    typed = body[body.index("if (uc_typed(cols.typed))"):body.index("} else {")]
    assert "slow" not in typed and "_tri(" not in typed.replace("str_tri(", "")   # plain booleans; two-slot startsWith keeps str_tri
    assert typed.count("const bool t") == 26


def _table(conds):
    rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}} for i, e in enumerate(conds)]
    pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "doc", "version": "default", "rules": rules}}
    return flatten(build_rule_table([pol]))


def test_a_slot_of_two_types_gets_no_typed_branch():
    one = hostsim.generate_uc(_table(['P.attr.x == "a"', "P.attr.y > 3"]).blob)[0]
    two = hostsim.generate_uc(_table(['P.attr.x == "a"', "P.attr.x > 3"]).blob)[0]
    assert "if (uc_typed(cols.typed))" in one
    assert two and "cols.typed" not in two and "r.typed" not in two


def test_list_equality_keeps_the_tri_state_terms(tmp_path):
    """`==` over two list slots compares containers, which only the tri-state terms can (they defer it): the table gets
    no typed branch, and its generated unit compiles and decides like oracle #2"""
    ft = _table(['"a" in P.attr.g', '"b" in R.attr.h', "P.attr.g == R.attr.h", 'P.attr.x == "q"'])
    src = hostsim.generate_uc(ft.blob)[0]
    assert src and "cols.typed" not in src
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    r = random.Random(77)
    lists = [[], ["a"], ["b"], ["a", "b"], ["b", "a"], ["a", 1]]
    reqs = [{"requestId": str(i), "actions": [f"a{j}" for j in range(4)],
             "principal": {"id": "p", "roles": ["user"], "attr": {"g": r.choice(lists), "x": r.choice(["q", "r"])}},
             "resource": {"kind": "doc", "id": f"r{i}", "attr": {"h": r.choice(lists)}}} for i in range(500)]
    b = Encoder(ft.manifest).encode(reqs)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for mode in (4, 5):
        assert (hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode) == want).all(), mode


# conditions whose negated literals turn an error into a different decision than a false: a guard that lets an
# empty list read at [0], a NaN, a mistyped or an absent value through changes the outcome
EDGE_CONDITIONS = ['!(P.attr.l[0] == "a")', '"a" in P.attr.l', "!(P.attr.n > 3)", "!(P.attr.n == 2)", '!(P.attr.s == "x")',
                   "!(R.attr.f == true)", "P.attr.n > 3 ? R.attr.f == true : P.attr.s == \"x\""]


def test_negated_literals_at_every_guard_edge(tmp_path):
    ft = _table(EDGE_CONDITIONS)
    src = hostsim.generate_uc(ft.blob)[0]
    assert "if (uc_typed(cols.typed))" in src
    assert re.search(r"typed_list\(r\.l\d+, 1u\)", src)   # l[0] is read: the guard needs one element
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    r = random.Random(5150)
    L = [[], ["a"], ["b", "a"], ["a", 2], ["x"] * 9, "a", None]
    N = [float("nan"), 1, 2, 5, -0.0, float("inf"), "5", True, None]
    S = ["x", "y", 3, None]
    F = [True, False, "true", 1, None]
    reqs = []
    for i in range(32 * 64):
        typed_lane = i % 32 < 16   # half of every warp well-typed, half at an edge
        p = {"l": r.choice(L[1:3]) if typed_lane else r.choice(L), "n": r.choice(N[1:6]) if typed_lane else r.choice(N),
             "s": r.choice(S[:2]) if typed_lane else r.choice(S)}
        res = {"f": r.choice(F[:2]) if typed_lane else r.choice(F)}
        reqs.append({"requestId": str(i), "actions": [f"a{j}" for j in range(len(EDGE_CONDITIONS))],
                     "principal": {"id": "p", "roles": ["user"], "attr": {k: v for k, v in p.items() if v is not None}},
                     "resource": {"kind": "doc", "id": f"r{i}", "attr": {k: v for k, v in res.items() if v is not None}}})
    b = Encoder(ft.manifest).encode(reqs)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for mode in (4, 5):
        assert (hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode) == want).all(), mode


# every edge of the guard, per attribute: absent, mistyped, NaN, signed zeros, infinities, lists it cannot hold
NUM_EDGES = [None, "5", True, float("nan"), 0.0, -0.0, float("inf"), float("-inf"), ["eng"]]
STR_EDGES = [None, 3, 2.5, True, False, ["eng"], {"a": "b"}]
LIST_EDGES = [None, [], ["eng", 3], ["eng", True], [f"g{i}" for i in range(1, 10)], ["eng"] + [f"g{i}" for i in range(1, 12)], "eng", 4]
BOOL_EDGES = [None, "true", 1, 0.0]
EDGES = {("principal", "email"): STR_EDGES, ("principal", "name"): STR_EDGES, ("principal", "groups"): LIST_EDGES,
         ("principal", "level"): NUM_EDGES, ("principal", "region"): STR_EDGES, ("resource", "prefix"): STR_EDGES,
         ("resource", "allowed_groups"): LIST_EDGES, ("resource", "team"): STR_EDGES, ("resource", "min_level"): NUM_EDGES,
         ("resource", "tier"): STR_EDGES, ("resource", "public"): BOOL_EDGES, ("resource", "owner"): STR_EDGES}


def _perturbed_inputs(w, n, seed):
    """C3 requests; about half of them (at random, so every warp mixes typed and perturbed lanes) get one to three
    attributes set to a guard edge, every edge of every attribute taken in turn"""
    r = random.Random(seed)
    reqs = w.inputs(w.fields(n), range(n))
    edges = [(k, v) for k, vs in EDGES.items() for v in vs]
    j = 0
    for q in reqs:
        if r.random() < 0.5:
            continue
        for _ in range(r.randrange(1, 4)):
            (who, name), v = edges[j % len(edges)]
            j += 1
            attrs = q[who]["attr"] if who == "principal" else q["resource"]["attr"]
            if v is None:
                attrs.pop(name, None)
            else:
                attrs[name] = list(v) if isinstance(v, list) else v
    return reqs


def _nan_inputs(w, n):
    """C3 requests where lanes 0..7 of every warp hold a NaN level and a public resource, lanes 8..11 a NaN min_level:
    a NaN ordering is an error, so `level > 5 ? tier == "gold" : public == true` (and its negation) does not hold,
    where a false ordering would take the `public` arm"""
    reqs = w.inputs(w.fields(n), range(n))
    for i, q in enumerate(reqs):
        if i % 32 < 8:
            q["principal"]["attr"]["level"] = float("nan")
            q["resource"]["attr"]["public"] = True
        elif i % 32 < 12:
            q["resource"]["attr"]["min_level"] = float("nan")
    return reqs


def _batches(n=4096):
    w, ft = _c3()
    enc = Encoder(ft.manifest)
    plain = enc.encode(w.inputs(w.fields(n), range(n)))
    mixed = enc.encode(_perturbed_inputs(w, n, 4521))
    nan = enc.encode(_nan_inputs(w, n))
    return ft, plain, mixed, nan


def _typed_lanes(b):
    """per request: every C3 slot holds the type its guard tests (a list slot: any list)"""
    slots = np.asarray(b.columns[3]).view(np.uint64).reshape(-1, b.n)
    top = slots >> np.uint64(48)
    string, boolean, lst = 0xFFF3, 0xFFF2, 0xFFF4
    ok = np.ones(b.n, dtype=bool)
    for v in C3_TYPES["typed_str"]:
        ok &= (slots[v] >> np.uint64(32)) == np.uint64(string << 16)
    for v in C3_TYPES["typed_num"]:
        ok &= ((top[v] & np.uint64(0xFFF0)) != np.uint64(0xFFF0)) & ~np.isnan(slots[v].view(np.float64))
    ok &= top[9] == np.uint64(boolean)
    for v in C3_LISTS:
        ok &= top[v] == np.uint64(lst)
    return ok


def test_c3_typed_and_perturbed_lanes_against_oracle(tmp_path):
    ft, plain, mixed, nan = _batches()
    assert _typed_lanes(plain).all()
    lanes = _typed_lanes(mixed).reshape(-1, 32)
    assert (lanes.any(axis=1) & ~lanes.all(axis=1)).all()   # every warp mixes the two branches
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    for b in (plain, mixed, nan):
        want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
        for mode in (4, 5):
            assert (hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode) == want).all(), mode
        if b is plain:
            assert hostsim.deferred(lib) == 0


def test_perturbed_values_reach_every_edge():
    w, _ = _c3()
    reqs = _perturbed_inputs(w, 4096, 4521)
    seen = set()
    for q in reqs:
        for (who, name), vs in EDGES.items():
            attrs = q[who]["attr"] if who == "principal" else q["resource"]["attr"]
            if name not in attrs:
                seen.add((who, name, "absent"))
                continue
            x = attrs[name]
            for k, v in enumerate(vs):
                same = (isinstance(v, float) and isinstance(x, float) and (math.isnan(v) and math.isnan(x) or (v == x and math.copysign(1, v) == math.copysign(1, x))))
                if same or (type(x) is type(v) and not isinstance(v, float) and x == v):
                    seen.add((who, name, k))
    for (who, name), vs in EDGES.items():
        for k, v in enumerate(vs):
            assert (who, name, "absent" if v is None else k) in seen, (who, name, v)


@pytest.mark.gpu
def test_c3_typed_and_perturbed_lanes_gpu():
    from cerbos_b200 import capi
    from cerbos_b200.device import DeviceBatch
    ft, plain, mixed, nan = _batches()
    ctx = capi.Context(0)
    try:
        t = ctx.load_table(ft.blob)
        specialised, note = t.wait_ready()
        assert specialised, note
        for b in (plain, mixed, nan):
            want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
            db = DeviceBatch(b, "cuda:0")
            db.run(t, 0)
            ctx.sync()
            cfg = ctx.last_kernel_config()
            assert cfg["unique_conditions"] and cfg["table_specialised"], cfg
            got = np.where(want != 0, db.effects(), 0)
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, bad[:8].tolist()
            assert (t.check(b.columns, b.n, b.max_actions, 0) == want).all()
        t.release()
    finally:
        ctx.close()
