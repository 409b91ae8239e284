"""Rule outputs (RuleRow.emit_output, ruletable.go:1065-1106): the output walk of the kernel core (cb::eval_request_outputs,
the body of check_outputs_kernel behind cgpu_check_outputs) against oracle #1 -- goldens, random policy sets, effect
neutrality, unlowered entries, record overflow -- and the host decoder (cerbos_b200/outputs.py) against oracle #1's
conversion.  The GPU tests run the same through Engine.check(include_outputs=True)."""
import copy
import json
import random
import struct

import numpy as np
import pytest

import fuzzgen
from cerbos_b200 import meta as M
from cerbos_b200 import outputs as O
from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table import layout as L
from cerbos_b200.table.flatten import flatten
from helpers import check_resources_api_outputs, engine_decisions, load_golden
from hostsim import driver as hostsim
from hostsim import outputs as hout
from oracle.celeval import CelMap, Duration, Timestamp, UInt, parse_timestamp
from oracle.check import CheckOracle, to_json_value

G = {"environment": "test"}
NOW = parse_timestamp("2024-01-01T00:00:00Z")
SEEDS = list(range(40))


def _store_docs():
    return [e["policy"] for e in load_golden("store_policies.json")]


def _strip_outputs(docs):
    docs = copy.deepcopy(docs)
    for d in docs:
        for kind in ("resourcePolicy", "principalPolicy"):
            for rule in (d.get(kind) or {}).get("rules") or []:
                rule.pop("output", None)
                for act in rule.get("actions") or []:
                    if isinstance(act, dict):
                        act.pop("output", None)
    return docs


def _kernel_outputs(ft, inputs, lenient=False, stride=4096, now=NOW):
    """-> (effects, action words, request records, [[entry, ...] per input], status) from the host build of the output walk."""
    enc = Encoder(ft.manifest, lenient_scope_search=lenient)
    b = enc.encode(inputs)
    fl = L.BATCH_FLAG_LENIENT if lenient else 0
    eff, am, rm, rec, st = hout.check_outputs(ft.blob, b.columns, b.n, b.max_actions, stride, now.ns, fl)
    outs = O.decode(rec, stride, ft.manifest, [inp.get("actions") or [] for inp in inputs]) if st == 0 else None
    return b, eff, am, rm, outs, st


def _meta_of(ft, b, lenient, now=NOW):
    return hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, now.ns, L.BATCH_FLAG_LENIENT if lenient else 0)


def _key(o):
    return (o["src"], o["action"], json.dumps(o["val"], sort_keys=True))


@pytest.fixture(scope="module")
def store():
    rt = build_rule_table(_store_docs())
    return rt, flatten(rt, globals_=G)


def test_store_table_declares_its_outputs(store):
    _rt, ft = store
    meta = np.frombuffer(ft.sections["META"].tobytes(), dtype=np.uint32)
    assert meta[L.META["n_output_rows"]] == len(ft.sections["OUT_ENTRIES"]) > 0
    assert meta[L.META["n_unlowered_outputs"]] == 1
    assert [(u["policy"], u["rule"]) for u in ft.manifest["unlowered_outputs"]] == [("resource.example.vdefault", "rule-001")]
    assert "resource.equipment_request.vdefault/acme#rule-001" in ft.manifest["output_sources"]


def test_table_without_outputs_has_no_output_sections(store):
    ft = flatten(build_rule_table(_strip_outputs(_store_docs())), globals_=G)
    meta = np.frombuffer(ft.sections["META"].tobytes(), dtype=np.uint32)
    assert "ROW_OUT" not in ft.sections and "output_sources" not in ft.manifest
    assert meta[L.META["n_output_rows"]] == meta[L.META["n_unlowered_outputs"]] == 0


def test_outputs_on_engine_goldens(store):
    """All 166 engine decisions: outputs equal oracle #1's as ordered lists and the goldens' as multisets; effects and
    metadata equal the metadata body's."""
    rt, ft = store
    orc = CheckOracle(rt, globals_=G)
    n = n_out = 0
    for cid, lenient, inp, want in engine_decisions():
        b, eff, am, rm, outs, st = _kernel_outputs(ft, [inp], lenient)
        if inp["resource"].get("kind") == "example":
            continue   # (the unlowered bare `R` output; test_unlowered_output)
        assert st == 0, cid
        py = orc.check(inp, NOW, lenient=lenient)
        assert outs[0] == py["outputs"], cid
        assert sorted(outs[0], key=_key) == sorted(want.get("outputs") or [], key=_key), cid
        e2, am2, rm2 = _meta_of(ft, b, lenient)
        assert (eff == e2).all() and (am == am2).all() and (rm == rm2).all(), cid
        n += len(inp["actions"])
        n_out += len(outs[0])
    assert n == 166 and n_out == 6


def test_outputs_on_api_goldens(store):
    rt, ft = store
    orc = CheckOracle(rt, globals_=G)
    n = 0
    for f, ci, want in check_resources_api_outputs():
        b, eff, am, rm, outs, st = _kernel_outputs(ft, [ci], now=NOW)
        assert st == 0, f
        assert outs[0] == orc.check(ci, NOW)["outputs"], f
        key = lambda o: (o["src"], o["action"])  # noqa: E731
        assert sorted(outs[0], key=key) == sorted(want, key=key), f
        e2, am2, rm2 = _meta_of(ft, b, False)
        assert (eff == e2).all() and (am == am2).all() and (rm == rm2).all(), f
        n += len(outs[0])
    assert n == 5


def test_outputs_leave_effects_and_metadata_alone_on_the_store(store):
    _rt, ft = store
    bare = flatten(build_rule_table(_strip_outputs(_store_docs())), globals_=G)
    for cid, lenient, inp, _want in engine_decisions():
        b, eff, am, rm, _outs, _st = _kernel_outputs(ft, [inp], lenient)
        b2 = Encoder(bare.manifest, lenient_scope_search=lenient).encode([inp])
        e2, am2, rm2 = _meta_of(bare, b2, lenient)
        assert (eff == e2).all() and (rm == rm2).all(), cid
        for k, a in enumerate(inp["actions"]):
            p, r = inp["principal"], inp["resource"]
            args = (p.get("id", ""), r.get("kind", ""), p.get("policyVersion") or "default", r.get("policyVersion") or "default")
            assert M.decode_action(int(am[0, k]), rm[0], ft.manifest, *args) == M.decode_action(int(am2[0, k]), rm2[0], bare.manifest, *args), (cid, a)


def _example_input(action):
    return {"requestId": "x", "actions": [action], "principal": {"id": "u", "roles": ["user"], "attr": {"ip": "10.20.1.1"}},
            "resource": {"kind": "example", "id": "e1", "attr": {}}}


def test_unlowered_output(store):
    """The store's `example` policy outputs the bare message `R`, which the device does not lower: the table builds, a
    request reaching the rule fails, one that does not succeeds, and the effect-only path still answers."""
    rt, ft = store
    rule = next(r for r in rt.rows if r.resource == "example" and r.emit_activated is not None)
    visiting, other = _example_input(rule.action), _example_input("zzz-not-an-action")
    *_r, st = _kernel_outputs(ft, [visiting])
    assert st & hout.STATUS_UNLOWERED
    _b, _e, _am, _rm, outs, st = _kernel_outputs(ft, [other])
    assert st == 0 and outs == [[]]
    b = Encoder(ft.manifest).encode([visiting])
    want = CheckOracle(rt, globals_=G).check(visiting, NOW)["actions"][rule.action]["effect"]
    assert hostsim.check(ft.blob, b.columns, b.n, b.max_actions, NOW.ns)[0, 0] == want


def test_record_overflow_reports_the_size_needed(store):
    rt, ft = store
    inputs = [ci for _f, ci, want in check_resources_api_outputs() if want]
    _b, _e, _am, _rm, full, st = _kernel_outputs(ft, inputs)
    assert st == 0
    b, _e, _am, _rm, _o, st = _kernel_outputs(ft, inputs, stride=16)
    assert st & hout.STATUS_OVERFLOW
    enc = Encoder(ft.manifest).encode(inputs)
    _e, _am, _rm, rec, _st = hout.check_outputs(ft.blob, enc.columns, enc.n, enc.max_actions, 16, NOW.ns)
    hdr = rec[:, :8].copy().view(np.uint32)
    assert (hdr[:, 1] == 0).all()                  # no partial entries
    need = int(hdr[:, 0].max())
    stride = (need + 7) // 8 * 8
    _b, _e, _am, _rm, again, st = _kernel_outputs(ft, inputs, stride=stride)
    assert st == 0 and again == full


# ---- the decoder against oracle #1's conversion ------------------------------------------------------------------------
def _enc_value(v) -> bytes:
    """A CEL value in the record form the device writes (layout.py OUT_TAGS)."""
    T = L.OUT_TAGS
    if v is None:
        return bytes([T["NULL"]])
    if isinstance(v, bool):
        return bytes([T["BOOL"], int(v)])
    if isinstance(v, UInt):
        return bytes([T["UINT"]]) + struct.pack("<Q", int(v))
    if isinstance(v, int):
        return bytes([T["INT"]]) + struct.pack("<q", v)
    if isinstance(v, float):
        return bytes([T["DOUBLE"]]) + struct.pack("<d", v)
    if isinstance(v, str):
        b = v.encode()
        return bytes([T["STRING"]]) + struct.pack("<I", len(b)) + b
    if isinstance(v, bytes):
        return bytes([T["BYTES"]]) + struct.pack("<I", len(v)) + v
    if isinstance(v, Timestamp):
        return bytes([T["TIMESTAMP"]]) + struct.pack("<q", v.ns)
    if isinstance(v, Duration):
        return bytes([T["DURATION"]]) + struct.pack("<q", v.ns)
    if isinstance(v, list):
        return bytes([T["LIST"]]) + struct.pack("<I", len(v)) + b"".join(_enc_value(x) for x in v)
    if isinstance(v, CelMap):
        return bytes([T["MAP"]]) + struct.pack("<I", len(v)) + b"".join(_enc_value(k) + _enc_value(x) for k, x in v.items())
    return bytes([T["NOT_CONVERTIBLE"]])


class _TypeValue:
    """Stands for a value with no google.protobuf.Value form (a CEL type)."""


_VALUES = [
    None, True, False, 0, -7, 2 ** 62, UInt(2 ** 64 - 1), 1.5, -0.0, 1e300, float("inf"), "", "héllo", b"", b"\x00\xffab",
    Timestamp(0), Timestamp(1_700_000_000_123_400_000), Timestamp(-1_000_000_001), Duration(0), Duration(90 * 10 ** 9),
    Duration(-1_500_000_000), Duration(1), [], [1, "a", [True, None]], CelMap([("k", 1), ("n", CelMap([("x", [1.25])]))]),
    CelMap([(1, "one"), (True, "t"), (UInt(3), "u")]), [_TypeValue()], CelMap([("t", _TypeValue())]), _TypeValue(),
]


@pytest.mark.parametrize("v", _VALUES, ids=lambda v: type(v).__name__)
def test_decoder_matches_oracle_conversion(v):
    rec = _enc_value(v)
    body = struct.pack("<HHI", 0, 0, 0) + rec
    record = struct.pack("<II", 8 + len(body), 1) + body
    got = O.decode_record(record, ["s#r"], ["view"])[0]["val"]
    try:
        want = to_json_value(v) if not isinstance(v, _TypeValue) else None
        if isinstance(v, _TypeValue):
            raise TypeError
    except Exception:
        want = O.NOT_CONVERTIBLE
    assert got == want


def test_decoder_reads_a_missing_value_as_none():
    record = struct.pack("<II", 17, 1) + struct.pack("<HHI", 0, 0, 0) + bytes([L.OUT_TAGS["NO_VALUE"]])
    assert O.decode_record(record, ["s#r"], ["view"]) == [{"src": "s#r", "action": "view", "val": None}]


# ---- differential fuzzing ----------------------------------------------------------------------------------------------
_OUT_EXPRS = [
    '"lit"', "P.id", "R.attr.dept", "R.attr.nope", "P.attr.level", "P.attr.level + 1", "P.attr.level * 2.5", "R.attr.allowed",
    "[P.id, R.id, 1, 2.5, true, null]", '{"a": P.attr.groups, "b": {"c": R.attr.public, "d": [1, [2, [3]]]}}', "now()",
    "runtime.effectiveDerivedRoles", '"x:%s".format([P.id])', "int(P.attr.level)", "uint(2)", 'b"\\x00ab"',
    'duration("90s")', 'timestamp("2024-02-03T04:05:06.5Z")', "type(P.id)", "[type(1)]", "{1: 2, true: 3}",
    "P.attr.groups.map(g, g + R.id)", "1 / 0", '{"k": 1 / 0}', "size(R.attr.allowed) > 1", "R.attr.size",
]


def _with_outputs(r: random.Random, docs):
    for d in docs:
        rules = (d.get("resourcePolicy") or {}).get("rules") or []
        for i, rule in enumerate(rules):
            rule["name"] = rule.get("name") or f"rule{i}"
            if r.random() < 0.7:
                when = {}
                if r.random() < 0.7:
                    when["ruleActivated"] = r.choice(_OUT_EXPRS)
                if r.random() < 0.6:
                    when["conditionNotMet"] = r.choice(_OUT_EXPRS)
                if when:
                    rule["output"] = {"when": when}
        for prule in (d.get("principalPolicy") or {}).get("rules") or []:
            for i, act in enumerate(prule["actions"]):
                act["name"] = f"p{i}"
                if r.random() < 0.6:
                    act["output"] = {"when": {"ruleActivated": r.choice(_OUT_EXPRS), "conditionNotMet": r.choice(_OUT_EXPRS)}}
        if rules and r.random() < 0.3:
            # a DENY ahead of an output row, and a rule whose several action patterns match one action
            rules.insert(0, {"name": "deny-first", "actions": ["edit"], "effect": "EFFECT_DENY", "roles": ["*"],
                             "condition": {"match": {"expr": "P.attr.vip == true"}}})
            rules.append({"name": "multi", "actions": ["edit", "*", "view"], "effect": "EFFECT_ALLOW", "roles": ["user", "*"],
                          "output": {"when": {"ruleActivated": '"multi-on"', "conditionNotMet": "R.attr.tier"}},
                          "condition": {"match": {"expr": "R.attr.public == true"}}})
    return docs


def _fuzz_case(seed):
    r = random.Random(seed)
    docs = _with_outputs(r, fuzzgen.rand_policies(r))
    rt = build_rule_table(docs)
    reqs = []
    for _ in range(24):
        q = fuzzgen.rand_request(r)
        if r.random() < 0.5:
            q["actions"] = r.sample(["edit", "view", "delete", "share:team"], r.randrange(1, 4))
        reqs.append(q)
    return docs, rt, flatten(rt), reqs


@pytest.mark.parametrize("seed", SEEDS)
def test_outputs_fuzz_against_oracle(seed):
    docs, rt, ft, reqs = _fuzz_case(seed)
    orc = CheckOracle(rt)
    b, eff, am, rm, outs, st = _kernel_outputs(ft, reqs)
    if st:   # only an unrepresentable run-time value may stop the call; find the request and check it alone
        assert st == hout.STATUS_UNSUPPORTED, st
    for i, q in enumerate(reqs):
        b1, e1, am1, rm1, o1, s1 = _kernel_outputs(ft, [q])
        if s1:
            assert s1 == hout.STATUS_UNSUPPORTED
            continue
        py = orc.check(q, NOW)
        assert o1[0] == py["outputs"], (seed, i)
        for k, a in enumerate(q["actions"]):
            assert int(e1[0, k]) == py["actions"][a]["effect"], (seed, i, a)
        if st == 0:
            assert outs[i] == o1[0], (seed, i)
    # effect neutral: the same policies without outputs give the same effects and metadata
    bare = flatten(build_rule_table(_strip_outputs(docs)))
    b2 = Encoder(bare.manifest).encode(reqs)
    e2, am2, rm2 = _meta_of(bare, b2, False)
    if st == 0:
        assert (eff == e2).all() and (rm == rm2).all()


def test_fuzz_covers_the_cases_that_matter():
    """The seeds reach principal-policy outputs, not-met entries, runtime.effectiveDerivedRoles and repeated visits."""
    seen = set()
    for seed in SEEDS:
        _docs, rt, ft, reqs = _fuzz_case(seed)
        orc = CheckOracle(rt)
        for q in reqs:
            outs = orc.check(q, NOW)["outputs"]
            if any(o["src"].startswith("principal.") for o in outs):
                seen.add("principal")
            if len({(o["src"], o["action"]) for o in outs}) < len(outs):
                seen.add("repeat")
            if any(o["val"] is None for o in outs):
                seen.add("no value")
            if any(o["val"] == O.NOT_CONVERTIBLE for o in outs):
                seen.add("not convertible")
    assert seen >= {"principal", "repeat", "no value", "not convertible"}, seen


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_engine_outputs_on_goldens_gpu():
    from cerbos_b200.engine import Engine
    docs = _store_docs()
    eng = Engine(docs, globals_=G)
    try:
        assert eng.has_outputs and [(u["policy"], u["rule"]) for u in eng.unlowered_outputs] == [("resource.example.vdefault", "rule-001")]
        orc = CheckOracle(build_rule_table(docs), globals_=G)
        for _cid, lenient, inp, _want in engine_decisions():
            if lenient or inp["resource"].get("kind") == "example":
                continue
            got = eng.check([inp], now_ns=NOW.ns, include_outputs=True)[0]
            py = orc.check(inp, NOW)
            assert got["outputs"] == py["outputs"]
            for a in inp["actions"]:
                assert got["actions"][a]["policy"] == py["actions"][a]["policy"]
        api = [ci for _f, ci, _w in check_resources_api_outputs()]
        got = eng.check(api, now_ns=NOW.ns, include_outputs=True)
        assert [g["outputs"] for g in got] == [orc.check(ci, NOW)["outputs"] for ci in api]
        from cerbos_b200.capi import CgpuError
        with pytest.raises(CgpuError):
            eng.check([_example_input("view")], now_ns=NOW.ns, include_outputs=True)
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS[:12])
def test_engine_outputs_fuzz_gpu(seed):
    from cerbos_b200.engine import Engine
    docs, rt, _ft, reqs = _fuzz_case(seed)
    orc = CheckOracle(rt)
    want = [orc.check(q, NOW) for q in reqs]
    eng = Engine(docs)
    try:
        from cerbos_b200.capi import CgpuError
        try:
            got = eng.check(reqs, now_ns=NOW.ns, include_outputs=True)
        except CgpuError:
            got = None
        if got is None:   # an unrepresentable value somewhere: every request alone
            for q, w in zip(reqs, want):
                try:
                    assert eng.check([q], now_ns=NOW.ns, include_outputs=True)[0]["outputs"] == w["outputs"]
                except CgpuError:
                    pass
        else:
            assert [g["outputs"] for g in got] == [w["outputs"] for w in want]
    finally:
        eng.close()


def _big_batch(n):
    r = random.Random(7)
    docs = _with_outputs(r, fuzzgen.rand_policies(random.Random(3)))
    _f, ci, _w = next((f, ci, w) for f, ci, w in check_resources_api_outputs() if w)
    store = _store_docs()
    reqs = [dict(ci, requestId=str(i), actions=["view", "create", "approve"][: 1 + i % 3]) for i in range(n)]
    return store, reqs, docs


@pytest.mark.gpu
def test_outputs_across_chunks_gpu():
    """A stride large enough that the output slab budget cuts the batch into several chunks: records come back
    index-aligned (each request's outputs carry its own id)."""
    from cerbos_b200 import capi
    store, reqs, _ = _big_batch(6000)
    for i, q in enumerate(reqs):
        q["principal"] = dict(q["principal"], id=f"p{i}")
    rt = build_rule_table(store)
    ft = flatten(rt, globals_=G)
    orc = CheckOracle(rt, globals_=G)
    ctx = capi.Context(0)
    try:
        t = ctx.load_table(ft.blob)
        b = Encoder(ft.manifest).encode(reqs)
        eff, am, rm, rec, need = t.check_outputs(b.columns, b.n, b.max_actions, 1 << 16, NOW.ns)
        assert need == 0
        got = O.decode(rec, 1 << 16, ft.manifest, [q["actions"] for q in reqs])
        for i in range(0, len(reqs), 97):
            assert got[i] == orc.check(reqs[i], NOW)["outputs"], i
        e2, am2, rm2 = t.check_meta(b.columns, b.n, b.max_actions, NOW.ns)
        assert (eff == e2).all() and (am == am2).all() and (rm == rm2).all()
        # too small a stride: fails, reports the size, and a retry with it gives the same records
        with pytest.raises(capi.CgpuError) as ei:
            t.check_outputs(b.columns, b.n, b.max_actions, 16, NOW.ns)
        stride = (ei.value.bytes_needed + 7) // 8 * 8
        assert 16 < stride <= 1 << 16
        *_p, rec2, need = t.check_outputs(b.columns, b.n, b.max_actions, stride, NOW.ns)
        assert need == 0 and O.decode(rec2, stride, ft.manifest, [q["actions"] for q in reqs]) == got
        t.release()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_outputs_two_devices_match_one_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("fewer than two GPUs")
    from cerbos_b200 import capi
    store, reqs, _ = _big_batch(20000)
    ft = flatten(build_rule_table(store), globals_=G)
    b = Encoder(ft.manifest).encode(reqs)
    res = []
    for n_dev in (1, 2):
        ctx = capi.Context(list(range(n_dev)))
        try:
            t = ctx.load_table(ft.blob)
            res.append(t.check_outputs(b.columns, b.n, b.max_actions, 1024, NOW.ns))
            t.release()
        finally:
            ctx.close()
    for x, y in zip(*res[:2]):
        assert np.array_equal(np.asarray(x), np.asarray(y))
