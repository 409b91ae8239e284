"""Table-specialised block evaluators (cerbos_b200/csrc/cb_specialize.h): the source the library hands to NVRTC at
table load is generated here for the workload / golden / fuzz tables, compiled for the host together with the kernel
core, and must give the oracles' bits.  (The GPU build of the same text is covered by tests/test_gpu_parity.py.)"""
import random

import numpy as np
import pytest

import workloads as W
from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table import layout as L
from cerbos_b200.table.flatten import flatten
from fuzzgen import rand_policies, rand_request
from hostsim import driver as hostsim
from oracle import cref


@pytest.mark.parametrize("name,n", [("C1", 1024), ("C2", 1 << 14), ("C3", 1 << 13)])
def test_workload_tables(name, n, tmp_path):
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    src = hostsim.generate(ft.blob)
    if name == "C3":
        assert src == "" or "spec_shape_0" in src    # 75 shapes: may exceed the code-size limits
    else:
        assert "struct SpecBlocks" in src
    if not src:
        pytest.skip("table does not qualify for specialisation")
    lib = hostsim.build_spec(ft.blob, str(tmp_path))
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for mode in (0, 3):   # global columns / staged column tiles
        got = hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode)
        assert (got == want).all(), mode


def test_generated_source_is_straight_line_for_c2():
    w = W.C2()
    _, ft, _ = W.build(w)
    src = hostsim.generate(ft.blob)
    assert src.count("spec_shape_") == 2 * 1 and src.count("term_lit(") == 4 and src.count("row_apply(") == 5   # one shape: 3 conditions / 4 terms, 5 rows
    assert "in_const_tri(cols.slot(" in src and "eq_tri(cols.slot(" in src                       # constants inlined as immediates
    assert all(f"case {k}:" in src for k in range(10))


@pytest.mark.parametrize("seed", range(12))
def test_random_tables(seed, tmp_path):
    r = random.Random(7000 + seed)
    # resource policies only (the lean body's domain): strip what the generator does not cover
    docs = [d for d in rand_policies(r) if "resourcePolicy" in d or "derivedRoles" in d or "exportVariables" in d or "exportConstants" in d]
    rt = build_rule_table(docs)
    ft = flatten(rt)
    src = hostsim.generate(ft.blob)
    if not src:
        pytest.skip("a condition has no flat form")
    lib = hostsim.build_spec(ft.blob, str(tmp_path))
    enc = Encoder(ft.manifest)
    inputs = [rand_request(r) for _ in range(300)]
    b = enc.encode(inputs)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, 0, 0)
    valid = want != 0
    for mode in (0, 3):
        got = hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode)
        assert (got[valid] == want[valid]).all(), (seed, mode)


# ---- unique-condition form (cb_uc.h image + cb::eval_request_uc; cb_specialize.h: generate_uc) -------------------------
@pytest.mark.parametrize("name,n", [("C2", 1 << 13), ("C3", 1 << 13)])
def test_unique_condition_body_on_workloads(name, n, tmp_path):
    """Generic condition evaluator (modes 4 / 5: rows from the image / merged records) and the generated straight-line
    evaluator, both against the oracle."""
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for mode in (4, 5):
        assert (hostsim.check(ft.blob, b.columns, b.n, b.max_actions, mode=mode) == want).all(), mode
    src, nu = hostsim.generate_uc(ft.blob)
    assert nu == {"C2": 3, "C3": 39}[name] and "struct SpecConds" in src
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    for mode in (4, 5):
        assert (hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode) == want).all(), mode


def test_unique_condition_source_shares_terms_for_c3():
    w = W.C3()
    _, ft, _ = W.build(w)
    src, nu = hostsim.generate_uc(ft.blob)
    # 39 distinct conditions over 26 distinct terms; every slot the table reads is loaded once into a register
    assert src.count("const int q") == 26 and src.count("// distinct condition") == 39
    assert all(f"r.s{v} = c.slot({v}u);" in src for v in range(12))


def test_c5_conditions_become_leaf_programs(tmp_path):
    """C5: 73 distinct conditions (the REQUIRE_PARENTAL_CONSENT leaves double the 37 trees as none(...)), 50 of them
    without a flat form.  Their bytecode is translated to straight-line code: 12 distinct leaves (atoms) shared by all
    the trees, rows in index form (more than 63 conditions).  Bit-exact against the oracle, and the specialised body
    decides the requests itself (nothing but the differing-version / unsupported cases may defer)."""
    w = W.C5()
    _, ft, enc = W.build(w)
    src, nu = hostsim.generate_uc(ft.blob)
    assert nu == 73 and src.count("CB_HD bool uc_atom_") == 12 and "kForm = CB_UC_FORM_INDEX" in src and "kPrograms = true" in src
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    b = w.columns(w.fields(4096), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for mode in (4, 5):
        assert (hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, mode=mode) == want).all(), mode
        assert hostsim.deferred(lib) == 0
    # the generic unique-condition body cannot evaluate programs: it defers, the general body answers
    assert (hostsim.check(ft.blob, b.columns, b.n, b.max_actions, mode=4) == want).all()
    assert hostsim.deferred() > b.n // 2


@pytest.mark.parametrize("seed", range(20))
def test_unique_condition_body_on_random_tables(seed, tmp_path):
    """Random policy sets x random requests: the generic unique-condition body and the generated evaluator -- flat terms,
    leaf programs translated from bytecode, leaf programs over one string slot evaluated by the per-string pre-pass --
    against oracle #2."""
    r = random.Random(9100 + seed)
    docs = [d for d in rand_policies(r) if "resourcePolicy" in d or "derivedRoles" in d or "exportVariables" in d or "exportConstants" in d]
    rt = build_rule_table(docs)
    ft = flatten(rt)
    lenient = seed % 4 == 0
    fl = L.BATCH_FLAG_LENIENT if lenient else 0
    enc = Encoder(ft.manifest, lenient_scope_search=lenient)
    inputs = [rand_request(r) for _ in range(300)]
    b = enc.encode(inputs)
    try:
        want = cref.check(ft.blob, b.columns, b.n, b.max_actions, 0, fl)
    except RuntimeError as e:
        if "-2" in str(e):
            pytest.skip("a request produces a run-time value outside the device's exact range (oracle #2 flags it too)")
        raise
    valid = want != 0
    try:
        got = hostsim.check(ft.blob, b.columns, b.n, b.max_actions, 0, fl, mode=4)
    except RuntimeError as e:
        if "-3" in str(e):
            pytest.skip("no unique-condition image (too many distinct conditions)")
        raise
    assert (got[valid] == want[valid]).all(), seed
    got = hostsim.check(ft.blob, b.columns, b.n, b.max_actions, 0, fl, mode=5)
    assert (got[valid] == want[valid]).all(), seed
    src, nu = hostsim.generate_uc(ft.blob)
    if src:
        lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
        got = hostsim.check_spec(lib, ft.blob, b.columns, b.n, b.max_actions, 0, fl, mode=5)
        assert (got[valid] == want[valid]).all(), seed


# ---- leaf programs (cb_specialize.h: translate_program / atom_source) on the reference's golden CEL expressions -----------
def _golden_leaf_cases():
    from test_table_oracles import _cel_cases
    groups = {}
    for f, e, req in _cel_cases():
        groups.setdefault(f, (req, []))[1].append(e)
    return groups


def test_leaf_programs_on_golden_expressions(tmp_path):
    """Every golden CEL leaf whose program the translator accepts (all but the ones building lists / maps in the arena)
    is evaluated by the generated straight-line code, inside tables of up to 16 rules, and must give oracle #1's
    answer -- the same bar the interpreter is held to in test_table_oracles.py."""
    from cerbos_b200.table.bytecode import Unsupported
    from oracle.celeval import parse_timestamp
    from oracle.check import CheckOracle
    now = parse_timestamp("2021-04-22T10:05:20.021-05:00")
    translated = checked = 0
    for gi, (f, (req, exprs)) in enumerate(sorted(_golden_leaf_cases().items())):
        inp = {"principal": dict(req.get("principal") or {}), "resource": dict(req.get("resource") or {})}
        if "auxData" in req:
            inp["auxData"] = req["auxData"]
        inp["resource"]["kind"] = "leave_request"
        inp["principal"].setdefault("roles", ["r"])

        def table(es):
            rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}} for i, e in enumerate(es)]
            pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "leave_request", "version": "default", "rules": rules}}
            rt = build_rule_table([pol])
            return rt, flatten(rt)

        ok = []
        for e in dict.fromkeys(exprs):
            try:
                _, ft1 = table([e])
            except Exception:
                continue          # not lowered at all (SPIFFE ...): rejected at table build
            src, _ = hostsim.generate_uc(ft1.blob)
            if "CB_HD bool uc_atom_" in src:
                ok.append(e)      # no flat form, and the translator takes its program
        translated += len(ok)
        for c0 in range(0, len(ok), 16):
            es = ok[c0:c0 + 16]
            rt, ft = table(es)
            src, _ = hostsim.generate_uc(ft.blob)
            assert src.count("CB_HD bool uc_atom_") >= 1
            d = tmp_path / f"g{gi}_{c0}"
            d.mkdir()
            lib = hostsim.build_spec(ft.blob, str(d), uc=True)
            one = dict(inp, actions=[f"a{i}" for i in range(len(es))])
            b = Encoder(ft.manifest).encode([one])
            want = CheckOracle(rt).check(one, now)["actions"]
            try:
                got = hostsim.check_spec(lib, ft.blob, b.columns, 1, b.max_actions, now.ns, mode=4)
            except RuntimeError as x:
                assert "-2" in str(x), (f, x)     # a run-time value outside the device's exact range: flagged, never wrong
                continue
            for i, e in enumerate(es):
                assert got[0, i] == want[f"a{i}"]["effect"], (f, e)
                checked += 1
    assert translated >= 60 and checked >= 50, (translated, checked)


# ---- the fuzz families of tests/fuzz_values.py through the generated leaf programs ------------------------------------------------
@pytest.mark.parametrize("family", ["time", "core", "math", "ip"])
def test_value_families_through_leaf_programs(family, tmp_path):
    """Random typed expressions (timestamps / durations, core semantics, ext.Math, inIPAddrRange) whose programs the translator
    takes, each with its negation, in one table; the generated straight-line code (host build) against oracle #1 on requests
    whose attributes change type.  (The interpreter's run over the same families is tests/test_fuzz_values.py.)"""
    import fuzz_values as FV
    from oracle.celeval import parse_timestamp
    from oracle.check import CheckOracle
    from test_fuzz_values import _table
    gen, req = {"time": (FV.TB, FV.rand_time_request), "core": (FV.CB, FV.rand_core_request), "math": (FV.M, FV.rand_request),
                "ip": (FV.IPB, FV.rand_ip_request)}[family]
    now = parse_timestamp("2024-03-10T06:59:59.5Z")
    r = random.Random(91000)
    es, tries = [], 0
    while len(es) < 8 and tries < 400:
        tries += 1
        e = gen(r)
        try:
            _, ft1 = _table([e])
        except Exception:  # noqa: BLE001 -- a construct the table build refuses: drawn again
            continue
        if "CB_HD bool uc_atom_" in hostsim.generate_uc(ft1.blob)[0]:
            es.append(e)
    assert len(es) >= 4
    es = es + [f"!({e})" for e in es]
    rt, ft = _table(es)
    src, _ = hostsim.generate_uc(ft.blob)
    assert src.count("CB_HD bool uc_atom_") >= 4
    lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
    orc, enc = CheckOracle(rt), Encoder(ft.manifest)
    compared = 0
    for _ in range(40):
        inp = dict(req(r), actions=[f"a{i}" for i in range(len(es))])
        want = orc.check(inp, now)["actions"]
        b = enc.encode([inp])
        try:
            got = hostsim.check_spec(lib, ft.blob, b.columns, 1, b.max_actions, now.ns, mode=4)
        except RuntimeError as x:
            assert "-2" in str(x), x          # a value outside the device's exact range: the call fails loudly
            continue
        for i, e in enumerate(es):
            assert got[0, i] == want[f"a{i}"]["effect"], (e, inp["principal"]["attr"], inp["resource"]["attr"])
            compared += 1
    assert compared >= 200
