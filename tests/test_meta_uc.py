"""Decision metadata from the unique-condition kernels (cb::eval_request_uc_meta, check_uc_meta / cb_spec_uc_meta*): the three
planes -- effect bytes, action words (policy, scope) and request records (first scopes, effectiveDerivedRoles) -- must be
byte for byte those of the reference-order metadata body (cb::eval_request_meta, hostsim.check_meta), on the workload
tables, on random resource-policy tables and on hand-built tables that probe where the bit-parallel walk and the reference's
own loop order part: how far effectiveDerivedRoles reaches along the scope chain, scopes whose ALLOWs do not count, kinds
with policies at some scopes only, unknown and missing roles, the row-range walk, lenient scope search, and the requests the
metadata form leaves to the reference-order body.  The hand-built tables are also decoded and held against oracle #1."""
import random

import numpy as np
import pytest

import workloads as W
from cerbos_b200 import meta as M
from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table import layout as L
from cerbos_b200.table.flatten import flatten
from fuzzgen import rand_policies, rand_request
from hostsim import driver as hostsim
from hostsim import meta_uc
from oracle.celeval import parse_timestamp
from oracle.check import CheckOracle
from test_uc_shapes import CASES as SHAPE_CASES, Case, _case as _shape_case, _request, _rp, _rule
from test_uc_walk import _case as _walk_case

NOW_NS = parse_timestamp("2024-01-01T00:00:00Z").ns
_built = {}


def _workload(name):
    if name not in _built:
        w = W.WORKLOADS[name]()
        _built[name] = (w, *W.build(w))
    return _built[name]


def _same(a, b, what):
    for x, y, plane in zip(a, b, ("effects", "action words", "request records")):
        assert x.shape == y.shape, (what, plane)
        bad = np.nonzero((x != y).reshape(len(x), -1).any(axis=1))[0]
        assert bad.size == 0, (what, plane, bad[:8].tolist())


def _oracle1(rt, ft, inputs, planes, lenient=False):
    """the decoded planes against oracle #1, request by request"""
    eff, am, rm = planes
    orc = CheckOracle(rt, lenient_scope_search=lenient)
    for j, inp in enumerate(inputs):
        py = orc.check(inp)
        p, rs = inp["principal"], inp["resource"]
        for k, a in enumerate(inp["actions"]):
            pol, sc = M.decode_action(int(am[j, k]), rm[j], ft.manifest, p.get("id", ""), rs.get("kind", ""),
                                      p.get("policyVersion") or "default", rs.get("policyVersion") or "default")
            w = py["actions"][a]
            assert (int(eff[j, k]), pol, sc) == (w["effect"], w["policy"], w["scope"]), (j, a)
        assert M.decode_edr(int(rm[j]["effective_derived_roles"]), ft.manifest) == py["effectiveDerivedRoles"], j


def _host_both(c, tmp_path, spec=True):
    """meta_uc.check_meta_uc (generic conditions; generated ones too when `spec`) against hostsim.check_meta on Case c;
    -> the reference planes and the deferral counts"""
    want = hostsim.check_meta(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags)
    got = meta_uc.check_meta_uc(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags)
    assert meta_uc.took(), c.name
    _same(got, want, (c.name, "generic"))
    deferred = [meta_uc.deferred()]
    if spec:
        lib = meta_uc.build_spec(c.ft.blob, str(tmp_path))
        got = meta_uc.check_meta_uc(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, lib=lib)
        assert meta_uc.took(lib), c.name
        _same(got, want, (c.name, "specialised"))
        deferred.append(meta_uc.deferred(lib))
    return want, deferred


# ---- CPU: workload tables --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,spec,max_deferred", [("C3", False, 0), ("C3", True, 0), ("C5", True, 0.05)])
def test_workloads_host(name, spec, max_deferred, tmp_path):
    w, _, ft, enc = _workload(name)
    b = W.columns_parallel(w, 2048, 777, enc)
    want = hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, NOW_NS)
    lib = meta_uc.build_spec(ft.blob, str(tmp_path)) if spec else None
    got = meta_uc.check_meta_uc(ft.blob, b.columns, b.n, b.max_actions, NOW_NS, lib=lib)
    assert meta_uc.took(lib)
    _same(got, want, name)
    assert meta_uc.deferred(lib) <= max_deferred * b.n, meta_uc.deferred(lib)


# ---- CPU: random resource-policy tables ------------------------------------------------------------------------------------
def _resource_only(docs):
    """rand_policies without principal and role policies and without rules reading runtime.effectiveDerivedRoles"""
    out = []
    for d in docs:
        if "principalPolicy" in d or "rolePolicy" in d:
            continue
        if "resourcePolicy" in d:
            rules = [x for x in d["resourcePolicy"]["rules"] if "runtime.effectiveDerivedRoles" not in str(x.get("condition", ""))]
            if not rules:
                continue
            d = {**d, "resourcePolicy": {**d["resourcePolicy"], "rules": rules}}
        out.append(d)
    return out


def test_random_tables_host():
    took = 0
    for seed in range(48):
        r = random.Random(51000 + seed)
        docs = _resource_only(rand_policies(r))
        rt = build_rule_table(docs)
        ft = flatten(rt)
        lenient = seed % 4 == 0
        enc = Encoder(ft.manifest, lenient_scope_search=lenient)
        b = enc.encode([rand_request(r) for _ in range(200)])
        fl = L.BATCH_FLAG_LENIENT if lenient else 0
        want = hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, 0, fl)
        got = meta_uc.check_meta_uc(ft.blob, b.columns, b.n, b.max_actions, 0, fl)
        _same(got, want, seed)
        took += meta_uc.took() and meta_uc.deferred() < b.n
    assert took >= 30, took


# ---- CPU: hand-built tables ------------------------------------------------------------------------------------------------
API = "api.cerbos.dev/v1"


def _edr_docs(leaf_effect):
    """kind doc at the root scope (importing derived role `helper` of role user) and at scope `a` (no derived roles): at `a`,
    role admin is decided for action view (`leaf_effect`), role user is not and walks on to the root"""
    drs = {"apiVersion": API, "derivedRoles": {"name": "drs", "definitions": [
        {"name": "helper", "parentRoles": ["user"]},
        {"name": "owner", "parentRoles": ["user", "admin"], "condition": {"match": {"expr": "R.attr.owner == P.id"}}},
        {"name": "anyone", "parentRoles": ["*"], "condition": {"match": {"expr": "P.attr.level > 5"}}}]}}
    root = _rp("doc", [_rule(["view", "edit"], "A", derived=["helper"], expr="P.attr.level >= 3"), _rule(["edit"], "A", derived=["owner"])], drs=True)
    leaf = _rp("doc", [_rule(["view"], leaf_effect, roles=["admin"]), _rule(["edit"], "D", roles=["admin"], expr="R.attr.size > 15")], scope="a")
    other = _rp("img", [_rule(["view"], "A", roles=["user"])])   # a second block shape
    return [drs, root, leaf, other]


def _edr_inputs(r, n):
    out = []
    for i in range(n):
        roles = [["admin", "user"], ["user", "admin"], ["admin"], ["user"], ["ghost", "admin", "user"]][i % 5]
        out.append(_request(r, "doc" if i % 7 else "img", roles, r.choice([["view"], ["view", "edit"], ["edit", "view"]]), scope=r.choice(["a", "", "a"])))
    return out


def _consent_docs():
    """doc at a.b asks for parental consent: its ALLOWs are decided at a (or not at all); img has policies at the root only, so
    chains from a.b pass scopes without a block of the request's kind; vid has a policy at every scope of the chain"""
    return [_rp("doc", [_rule(["view"], "A", roles=["user"])]),
            _rp("doc", [_rule(["view", "edit"], "A", roles=["user"], expr="P.attr.level > 4")], scope="a"),
            _rp("doc", [_rule(["view", "edit"], "A", roles=["*"]), _rule(["edit"], "D", roles=["manager"])], scope="a.b", consent=True),
            _rp("img", [_rule(["view"], "A", roles=["manager"]), _rule(["edit"], "D", roles=["*"], expr='R.attr.dept == "d1"')]),
            _rp("vid", [_rule(["view"], "D", roles=["user"], expr="P.attr.vip == true")]),
            _rp("vid", [_rule(["edit"], "D", roles=["manager"], expr="P.attr.level < 2")], scope="a"),
            _rp("vid", [_rule(["view", "edit"], "A", roles=["user", "manager"])], scope="a.b")]


def _consent_inputs(r, n):
    return [_request(r, r.choice(["doc", "img", "vid"]), r.sample(["user", "manager", "ghost"], r.randrange(1, 3)), r.choice([["view"], ["view", "edit"]]),
                     scope=r.choice(["a.b", "a", "", "a.b"])) for _ in range(n)]


def _defer_inputs(r, n):
    """a third of the requests in a principal policy version the table lacks (versions differ: reference-order body)"""
    out = _consent_inputs(r, n)
    for inp in out[::3]:
        inp["principal"]["policyVersion"] = "v7"
    return out


HAND = {
    "edr_allow_leaf": lambda: Case("edr_allow_leaf", _edr_docs("A"), _edr_inputs(random.Random(61), 601)),
    "edr_deny_leaf": lambda: Case("edr_deny_leaf", _edr_docs("D"), _edr_inputs(random.Random(62), 601)),
    "consent_partial_kinds": lambda: Case("consent_partial_kinds", _consent_docs(), _consent_inputs(random.Random(63), 801)),
    "lenient": lambda: Case("lenient_meta", _consent_docs(), [_request(random.Random(64 + i), ["doc", "img", "vid"][i % 3], ["user", "manager"][: 1 + i % 2], ["view", "edit"],
                                                                       scope=["a.b.c.d", "a.q", "zz", "a.b", ""][i % 5]) for i in range(500)], lenient=True),
    "versions": lambda: Case("versions", _consent_docs(), _defer_inputs(random.Random(65), 600)),
}
_hand = {}


def _hand_case(name):
    if name not in _hand:
        _hand[name] = HAND[name]()
    return _hand[name]


@pytest.mark.parametrize("name", list(HAND))
def test_hand_built_host(name, tmp_path):
    c = _hand_case(name)
    want, deferred = _host_both(c, tmp_path)
    _oracle1(c.rt, c.ft, c.inputs, want, c.lenient)
    if name == "versions":
        assert all(d == len(c.inputs[::3]) for d in deferred), deferred
    else:
        assert deferred == [0, 0], deferred


def test_edr_reach_both_directions():
    """role admin decides view at scope a: an ALLOW there ends the reference's role loop before role user reaches the root,
    whose derived role `helper` (of role user) then stays out; a DENY does not, and `helper` is in"""
    for name, want_helper in (("edr_allow_leaf", False), ("edr_deny_leaf", True)):
        c = _hand_case(name)
        eff, am, rm = meta_uc.check_meta_uc(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags)
        hits = [j for j, inp in enumerate(c.inputs) if inp["resource"]["kind"] == "doc" and inp["resource"].get("scope") == "a"
                and inp["principal"]["roles"] == ["admin", "user"] and inp["actions"] == ["view"] and inp["principal"]["attr"]["level"] >= 3]
        assert len(hits) >= 5, name
        for j in hits:
            assert ("helper" in M.decode_edr(int(rm[j]["effective_derived_roles"]), c.ft.manifest)) == want_helper, (name, j)


def test_no_role_request():
    """a request without roles, where the encoder takes one: NO_MATCH words, no derived roles"""
    c = _hand_case("consent_partial_kinds")
    inp = _request(random.Random(66), "doc", [], ["view", "edit"], scope="a")
    try:
        b = c.enc.encode([inp] * 3)
    except Exception:   # an encoder that refuses a principal without roles leaves nothing to check
        pytest.skip("the encoder refuses requests without roles")
    want = hostsim.check_meta(c.ft.blob, b.columns, b.n, b.max_actions, 0, 0)
    got = meta_uc.check_meta_uc(c.ft.blob, b.columns, b.n, b.max_actions, 0, 0)
    _same(got, want, "no role")


@pytest.mark.parametrize("name", sorted(SHAPE_CASES) + ["walk:long_scope", "walk:same_pair"])
def test_shape_cases_host(name, tmp_path):
    """every table and batch shape the unique-condition kernels specialise on: condition-word forms (mask-32, mask-64, index),
    role-table widths, segment and row-range walks (long_scope: more than 16 rows per scope), global images, lists longer
    than the register cache holds (deferred by the generated conditions)"""
    c = _walk_case(name[5:]) if name.startswith("walk:") else _shape_case(name)
    _, deferred = _host_both(c, tmp_path, spec=name.startswith("walk:") or c.spec_host)
    if name == "lists_warp":
        assert deferred[1] > 0


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def _set_env(monkeypatch, env):
    for k in ("CERBOS_B200_NO_JIT", "CERBOS_B200_NO_STAGE", "CERBOS_B200_UC"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


class _Loaded:
    """a fresh context (it reads the environment switches) with `blob` loaded and its specialised kernels ready"""
    def __init__(self, blob):
        from cerbos_b200 import capi
        self.ctx = capi.Context(0)
        self.t = self.ctx.load_table(blob)
        self.specialised = self.t.wait_ready()[0]

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.t.release()
        self.ctx.close()


# (workload, environment, whether a unique-condition kernel takes the metadata): C5's conditions include programs, which only
# its specialised kernel evaluates, so without NVRTC its metadata stays on the reference-order body
GPU_RUNS = [("C3", {}, True), ("C5", {}, True), ("C3", {"CERBOS_B200_NO_JIT": "1"}, True), ("C5", {"CERBOS_B200_NO_JIT": "1"}, False),
            ("C3", {"CERBOS_B200_NO_STAGE": "1"}, True), ("C5", {"CERBOS_B200_NO_STAGE": "1"}, True), ("C2", {"CERBOS_B200_UC": "1"}, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,env,uc", GPU_RUNS, ids=[f"{n}-{'-'.join(e) or 'default'}" for n, e, _ in GPU_RUNS])
def test_workloads_gpu(name, env, uc, monkeypatch):
    """2^20 requests: the effect bytes of cgpu_check_meta equal cgpu_check's.  2^16 requests: all three planes equal the
    reference-order body of the host build, and the launch ran the unique-condition kernel where the table allows it."""
    _set_env(monkeypatch, env)
    w, _, ft, enc = _workload(name)
    with _Loaded(ft.blob) as L_:
        b = W.columns_parallel(w, 1 << 20, 0, enc)
        eff, _, _ = L_.t.check_meta(b.columns, b.n, b.max_actions, NOW_NS)
        assert L_.ctx.last_kernel_config()["unique_conditions"] == uc
        assert (eff == L_.t.check(b.columns, b.n, b.max_actions, NOW_NS)).all(), name
        b = W.columns_parallel(w, 1 << 16, 1 << 20, enc)
        got = L_.t.check_meta(b.columns, b.n, b.max_actions, NOW_NS)
        assert L_.ctx.last_kernel_config()["unique_conditions"] == uc
        _same(got, hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, NOW_NS), name)


@pytest.mark.gpu
def test_deferred_versions_gpu():
    """a C3 batch with a third of its requests in no resource policy version (CB_NONE16: a version the table lacks), so
    that it differs from the principal's: those go through the deferral list to the reference-order body"""
    w, _, ft, enc = _workload("C3")
    b = W.columns_parallel(w, 3 * 4096 + 77, 99, enc)
    cols = list(b.columns)
    h1 = np.array(cols[1], copy=True)
    h1.view(np.uint16).reshape(b.n, 4)[::3, 0] = 0xFFFF
    cols[1] = h1
    with _Loaded(ft.blob) as L_:
        before = L_.ctx.deferred_count()
        got = L_.t.check_meta(cols, b.n, b.max_actions, NOW_NS)
        assert L_.ctx.last_kernel_config()["unique_conditions"]
        assert L_.ctx.deferred_count() - before >= (b.n + 2) // 3
    _same(got, hostsim.check_meta(ft.blob, cols, b.n, b.max_actions, NOW_NS), "versions")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPE_CASES) + ["walk:long_scope"] + list(HAND))
def test_cases_gpu(name, monkeypatch):
    """the shape and hand-built cases through cgpu_check_meta on the unique-condition kernels"""
    _set_env(monkeypatch, {"CERBOS_B200_UC": "1"})
    c = _walk_case(name[5:]) if name.startswith("walk:") else _hand_case(name) if name in HAND else _shape_case(name)
    with _Loaded(c.ft.blob) as L_:
        got = L_.t.check_meta(c.b.columns, c.b.n, c.b.max_actions, 0, c.flags)
        assert L_.ctx.last_kernel_config()["unique_conditions"], name
    _same(got, hostsim.check_meta(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags), name)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_random_tables_gpu(seed, monkeypatch):
    _set_env(monkeypatch, {"CERBOS_B200_UC": "1"})
    r = random.Random(51000 + seed)
    docs = _resource_only(rand_policies(r))
    ft = flatten(build_rule_table(docs))
    lenient = seed % 4 == 0
    b = Encoder(ft.manifest, lenient_scope_search=lenient).encode([rand_request(r) for _ in range(2000)])
    fl = L.BATCH_FLAG_LENIENT if lenient else 0
    with _Loaded(ft.blob) as L_:
        got = L_.t.check_meta(b.columns, b.n, b.max_actions, 0, fl)
    _same(got, hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, 0, fl), seed)
