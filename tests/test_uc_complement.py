"""Complement-coded rows of the unique-condition image (cb_uc.h): a condition and its final negation -- a top-level `none`,
as the REQUIRE_PARENTAL_CONSENT scopes wrap their conditional ALLOWs -- share one base condition and one bit of the
condition word, and a row needs each of its conditions true or false.  Tables whose base conditions fit 31 bits take the
32-bit form even with 32..62 distinct conditions; tables with more base conditions keep one bit per distinct condition.

The negation is exact on one bit, errors included: a failed term is neither true nor false as a literal, so the
condition does not hold and its `none` does, as in the reference.  Requests with absent and mistyped attributes are
therefore decided in the kernel (nothing deferred) and must agree with oracle #2 (all requests) and oracle #1 (a sample),
through the generic and the generated evaluator, on the host and on the device; derived roles on a condition and on its
negation are checked in the metadata form against the reference-order body."""
import random
import re

import numpy as np
import pytest

from hostsim import driver as hostsim
from test_meta_uc import _Loaded, _host_both, _oracle1, _same, _set_env
from test_uc_shapes import Case, _check_oracle1, _rp, _rule

ROLES = ["user", "manager", "admin"]
ACTIONS = [f"a{i}" for i in range(6)]
# one scalar attribute per condition shape; requests make each absent or mistyped now and then
SHAPES = ["P.attr.level >= {k}", 'R.attr.dept == "d{k}"', "R.attr.size < {k} || P.attr.vip == true", "P.attr.dept == R.attr.dept && R.attr.size > {k}",
          "R.attr.owner == P.id || P.attr.level > {k}", '!(R.attr.tier == "t{k}")']


def _conds(n):
    """n distinct conditions with a flat (DNF) form"""
    return [SHAPES[i % len(SHAPES)].format(k=i % 7) + ("" if i < len(SHAPES) else f" || R.attr.size == {100 + i}") for i in range(n)]


def _attrs(r):
    p = {"dept": f"d{r.randrange(7)}", "level": r.randrange(8), "vip": r.random() < 0.2}
    res = {"dept": f"d{r.randrange(7)}", "size": r.randrange(9), "owner": r.choice(["alice", "bob"]), "tier": f"t{r.randrange(7)}"}
    # about a third of the requests: one or two attributes absent or a scalar of a type their comparison does not take (an
    # error; lists and maps are left out: the tri-state terms defer containers whatever the image's form)
    for _ in range(r.choice([0, 0, 0, 0, 1, 2])):
        who, k = r.choice([(p, "level"), (p, "vip"), (p, "dept"), (res, "dept"), (res, "size"), (res, "owner"), (res, "tier")])
        bad = r.choice([None, "7", True, 3.5, "d1"])
        if bad is None:
            who.pop(k, None)
        else:
            who[k] = bad
    return p, res


def _inputs(r, kinds, scopes, n):
    out = []
    for _ in range(n):
        p, res = _attrs(r)
        out.append({"requestId": "u", "actions": r.sample(ACTIONS, r.randrange(1, len(ACTIONS) + 1)),
                    "principal": {"id": r.choice(["alice", "bob", "carol"]), "roles": r.sample(ROLES, r.randrange(1, 3)), "attr": p},
                    "resource": {"kind": r.choice(kinds), "id": "x", "scope": r.choice(scopes), "attr": res}})
    return out


def _consent_docs(r, conds, n_kinds, consent_from=0, drs=None):
    """per kind: a root policy, a REQUIRE_PARENTAL_CONSENT policy at scope a and a plain one at a.b.  The root rules use
    conds[consent_from:] as they are; the consent scope's conditional ALLOWs use conds[:n] (they become DENY rows on their
    negations), so that conds[consent_from:n] occur both ways"""
    docs = []
    if drs:
        docs.append({"apiVersion": "api.cerbos.dev/v1", "derivedRoles": {"name": "drs", "definitions": drs}})
    pos, neg = conds[consent_from:], conds
    for k in range(n_kinds):
        kind = f"k{k}"
        for scope, pool, consent in (("", pos, False), ("a", neg, True), ("a.b", pos, False)):
            rules = []
            for i in range(5):
                j = (k * 5 + i) % len(pool)
                eff = "D" if (i == 4 and not consent) else "A"
                if drs and i == 2:
                    rules.append(_rule(r.sample(ACTIONS, 2), eff, derived=[drs[(k + len(scope)) % len(drs)]["name"]], expr=pool[(j + 3) % len(pool)]))
                else:
                    rules.append(_rule(r.sample(ACTIONS, r.randrange(1, 4)), eff, roles=["*"] if i == 0 else r.sample(ROLES, 2), expr=pool[j]))
            doc = _rp(kind, rules, scope=scope, consent=consent, drs=bool(drs))
            docs.append(doc)
    return docs


def _form(src):
    m = re.search(r"// (\d+) distinct conditions on (\d+) base conditions", src)
    return re.search(r"kForm = CB_UC_FORM_(\w+)", src).group(1), (int(m.group(1)), int(m.group(2))) if m else None


def case_consent():
    """12 conditions, each with its negation from the consent scope: 24 distinct, 12 base"""
    r = random.Random(71)
    return Case("consent", _consent_docs(r, _conds(12), 6), _inputs(r, [f"k{k}" for k in range(6)], ["", "a", "a.b"], 4099), spec_host=True)


def case_fold62():
    """27 conditions and 28 negations: 55 distinct conditions (one bit each would need 64-bit masks), 28 base"""
    r = random.Random(72)
    return Case("fold62", _consent_docs(r, _conds(28), 12, consent_from=1), _inputs(r, [f"k{k}" for k in range(12)], ["", "a", "a.b"], 4101), spec_host=True)


def case_wide():
    """36 base conditions, 10 of them negated too: more base conditions than 31 bits, so one bit per distinct condition"""
    r = random.Random(73)
    conds = _conds(36)
    docs = _consent_docs(r, conds[:10], 2) + [_rp(f"w{k}", [_rule(r.sample(ACTIONS, 2), "DA"[i % 2], roles=r.sample(ROLES, 2), expr=conds[(4 * k + i) % 36])
                                                            for i in range(4)]) for k in range(9)]
    return Case("wide", docs, _inputs(r, ["k0", "k1"] + [f"w{k}" for k in range(9)], ["", "a", "a.b"], 3007), spec_host=True)


def case_drs():
    """derived roles on a condition and on its negation, rules on both, for the metadata form"""
    r = random.Random(74)
    conds = _conds(8)
    drs = [{"name": "owner", "parentRoles": ["user"], "condition": {"match": {"expr": conds[4]}}},
           {"name": "stranger", "parentRoles": ["user", "manager"], "condition": {"match": {"none": {"of": [{"expr": conds[4]}]}}}},
           {"name": "senior", "parentRoles": ["manager"], "condition": {"match": {"none": {"of": [{"expr": conds[0]}]}}}}]
    return Case("drs", _consent_docs(r, conds, 4, drs=drs), _inputs(r, [f"k{k}" for k in range(4)], ["", "a", "a.b"], 2051), spec_host=True)


CASES = {"consent": case_consent, "fold62": case_fold62, "wide": case_wide, "drs": case_drs}
# (kForm, (distinct, base) listed by the generator for a complement-coded image, None otherwise)
FORMS = {"consent": ("MASK32", (24, 12)), "fold62": ("MASK32", (55, 28)), "wide": ("MASK64", None), "drs": ("MASK32", (16, 8))}
_built = {}


def _case(name):
    if name not in _built:
        _built[name] = CASES[name]()
    return _built[name]


TYPES = {("principal", "level"): int, ("principal", "vip"): bool, ("principal", "dept"): str, ("resource", "dept"): str,
         ("resource", "size"): int, ("resource", "owner"): str, ("resource", "tier"): str}


def _errors(c):
    """requests with an absent or mistyped attribute"""
    return sum(any(type(inp[who]["attr"].get(k)) is not t for (who, k), t in TYPES.items()) for inp in c.inputs)


@pytest.mark.parametrize("name", list(CASES))
def test_form_and_decisions_host(name, tmp_path):
    """the form each table takes, and the generic (modes 4 / 5) and generated evaluators against oracle #2, nothing deferred"""
    c = _case(name)
    src, nu = hostsim.generate_uc(c.ft.blob)
    form, listed = _form(src)
    assert (form, listed) == FORMS[name], (name, form, listed, nu)
    if listed:
        # every distinct condition is one base condition, as itself or negated, and every base condition is used
        uses = re.findall(r"// distinct condition \d+: (!?)base condition (\d+)", src)
        assert len(uses) == len(set(uses)) == nu and {int(b) for _, b in uses} == set(range(1, listed[1] + 1))
        assert "val.lo |= (uint32_t)" in src and "val.hi |=" not in src
    if name == "fold62":
        assert 32 <= nu <= 62
    if name == "wide":
        assert nu == 46 and "base condition" not in src
    assert _errors(c) > c.b.n // 5, name
    want = c.want
    valid = want != 0
    assert 0.1 <= (want[valid] == 1).mean() <= 0.9, name
    _check_oracle1(c, want)
    lib = hostsim.build_spec(c.ft.blob, str(tmp_path), uc=True)
    for mode in (4, 5):
        got = hostsim.check(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body() == mode and hostsim.deferred() == 0, (name, mode)
        assert (got[valid] == want[valid]).all(), (name, mode)
        got = hostsim.check_spec(lib, c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body(lib) == mode and hostsim.deferred(lib) == 0, (name, mode)
        assert (got[valid] == want[valid]).all(), (name, mode)


def test_error_makes_the_negation_hold(tmp_path):
    """one base condition, its negation from the consent scope: a request whose attribute is absent or mistyped fails the
    condition, so the consent scope's DENY on the negation applies, exactly as for a false condition"""
    docs = [_rp("doc", [_rule(["view"], "A", roles=["user"], expr="P.attr.level >= 3")]),
            _rp("doc", [_rule(["view"], "A", roles=["user"], expr="P.attr.level >= 3")], scope="a", consent=True)]
    values = [5, 1, None, "5", True, [4], float("nan"), 3]
    inputs = [{"requestId": str(i), "actions": ["view"], "principal": {"id": "p", "roles": ["user"], "attr": {} if v is None else {"level": v}},
               "resource": {"kind": "doc", "id": "x", "scope": sc, "attr": {}}} for i, (v, sc) in enumerate((v, sc) for v in values for sc in ("", "a"))]
    c = Case("one", docs, inputs)
    assert _form(hostsim.generate_uc(c.ft.blob)[0]) == ("MASK32", (2, 1))
    want = c.want[:, 0]
    # root scope: ALLOW iff level >= 3; scope a: DENY unless level >= 3, then the root decides
    assert want.tolist() == [1 if isinstance(v, (int, float)) and not isinstance(v, bool) and v == v and v >= 3 else 2 for v in values for _ in (0, 1)]
    lib = hostsim.build_spec(c.ft.blob, str(tmp_path), uc=True)
    for mode in (4, 5):
        assert (hostsim.check(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, mode=mode)[:, 0] == want).all() and hostsim.deferred() == 0
        assert (hostsim.check_spec(lib, c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, mode=mode)[:, 0] == want).all() and hostsim.deferred(lib) == 0


def test_derived_roles_on_negations_meta_host(tmp_path):
    c = _case("drs")
    want, deferred = _host_both(c, tmp_path)
    assert deferred == [0, 0]
    edr = want[2]["effective_derived_roles"]
    assert len(set(edr.tolist())) >= 4   # owner / stranger / senior reached, in different combinations
    _oracle1(c.rt, c.ft, c.inputs[:300], tuple(p[:300] for p in want))


def test_no_negations_no_change():
    """a table without negated conditions keeps one bit per distinct condition"""
    r = random.Random(75)
    docs = [_rp(f"k{k}", [_rule(r.sample(ACTIONS, 2), "A", roles=["user"], expr=x) for x in _conds(10)[k::2]]) for k in range(2)]
    c = Case("plain", docs, _inputs(r, ["k0", "k1"], [""], 64))
    src, nu = hostsim.generate_uc(c.ft.blob)
    assert nu == 10 and _form(src) == ("MASK32", None) and "base condition" not in src


# ---- the device -----------------------------------------------------------------------------------------------------------
GPU_ENVS = [{}, {"CERBOS_B200_NO_JIT": "1"}, {"CERBOS_B200_NO_STAGE": "1"}]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_decisions_gpu(name, monkeypatch):
    """the NVRTC-specialised kernel, the ahead-of-time kernel (generic conditions) and the global-memory image, against
    oracle #2; device-resident batch and host-buffer path"""
    from cerbos_b200.device import DeviceBatch
    c = _case(name)
    want = c.want
    for env in GPU_ENVS:
        _set_env(monkeypatch, {"CERBOS_B200_UC": "1", **env})
        with _Loaded(c.ft.blob) as L_:
            assert L_.specialised == ("CERBOS_B200_NO_JIT" not in env), (name, env)
            d0 = L_.ctx.deferred_count()
            db = DeviceBatch(c.b, "cuda:0")
            db.run(L_.t, 0, c.flags)
            L_.ctx.sync()
            cfg = L_.ctx.last_kernel_config()
            assert cfg["unique_conditions"] and cfg["table_specialised"] == L_.specialised, (name, env, cfg)
            got = np.where(want != 0, db.effects(), 0)
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, (name, env, bad[:8].tolist())
            assert L_.ctx.deferred_count() == d0, (name, env)
            assert (L_.t.check(c.b.columns, c.b.n, c.b.max_actions, 0, c.flags) == want).all(), (name, env)


@pytest.mark.gpu
@pytest.mark.parametrize("env", GPU_ENVS, ids=["default", "no_jit", "no_stage"])
def test_derived_roles_on_negations_meta_gpu(env, monkeypatch):
    c = _case("drs")
    _set_env(monkeypatch, {"CERBOS_B200_UC": "1", **env})
    with _Loaded(c.ft.blob) as L_:
        got = L_.t.check_meta(c.b.columns, c.b.n, c.b.max_actions, 0, c.flags)
        assert L_.ctx.last_kernel_config()["unique_conditions"]
    _same(got, hostsim.check_meta(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags), "drs")
