"""Unique-condition kernels (cb_uc.h image, cb::eval_request_uc / cb::uc_walk) on every table and batch shape they
specialise on: one role column and more than four, 64-bit role words, index-form rows without leaf programs, scope chains
with REQUIRE_PARENTAL_CONSENT and kinds missing from a scope, lenient scope search, list operands of every length and
type inside one warp, and a global image too large for the merged-row pre-pass.

Every case is a resource-policy-only table (the lean domain) built here, and proves that it reached the branch it is
named after: on the host from the generated source and the body the host build ran, on the device from the launch
configuration.  Decisions are compared with oracle #2 (all requests) and oracle #1 (a sample)."""
import functools
import os
import random

import numpy as np
import pytest

from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table import layout as L
from cerbos_b200.table.flatten import flatten
from hostsim import driver as hostsim
from oracle import cref
from oracle.check import CheckOracle

API = "api.cerbos.dev/v1"
CONSENT = "SCOPE_PERMISSIONS_REQUIRE_PARENTAL_CONSENT_FOR_ALLOWS"
CHUNK = 4096
FORMS = {"CB_UC_FORM_MASK32": "mask32", "CB_UC_FORM_MASK64": "mask64", "CB_UC_FORM_INDEX": "index"}


# ---- policy and batch builder ------------------------------------------------------------------------------------------
def _rp(kind, rules, scope="", consent=False, drs=False):
    rp = {"resource": kind, "version": "default", "rules": rules}
    if scope:
        rp["scope"] = scope
    if consent:
        rp["scopePermissions"] = CONSENT
    if drs:
        rp["importDerivedRoles"] = ["drs"]
    return {"apiVersion": API, "resourcePolicy": rp}


def _rule(actions, effect, roles=None, derived=None, expr=None):
    r = {"actions": list(actions), "effect": "EFFECT_ALLOW" if effect == "A" else "EFFECT_DENY"}
    if roles:
        r["roles"] = list(roles)
    if derived:
        r["derivedRoles"] = list(derived)
    if expr:
        r["condition"] = {"match": {"expr": expr}}
    return r


def _flat_conds(n, salt=0):
    """n distinct conditions over scalar attributes, each with a flat (DNF) form, satisfied by part of the requests"""
    out = []
    for i in range(n):
        j = (i + salt) % 6
        out.append([f"P.attr.level >= {i % 10}", f'R.attr.dept == "d{i % 6}"', f"R.attr.size < {i % 20} || P.attr.vip == true",
                    f'P.attr.dept == R.attr.dept && R.attr.size > {i % 7}', f'"g{i % 8}" in P.attr.groups', f"R.attr.owner == P.id || P.attr.level > {i % 9}"][j]
                   + ("" if i < 6 else f" || R.attr.size == {100 + i}"))
    return out


def _attrs(r):
    p = {"dept": f"d{r.randrange(6)}", "level": r.randrange(10), "vip": r.random() < 0.2, "groups": [f"g{r.randrange(8)}" for _ in range(r.randrange(4))]}
    res = {"dept": f"d{r.randrange(6)}", "size": r.randrange(20), "owner": r.choice(["alice", "bob", "carol"])}
    return p, res


def _asets(r, actions, kmax, n=8):
    """a few fixed action lists (the merged rows of n_asets x n_rows stay small), one of them kmax long"""
    return [list(actions[:kmax])] + [r.sample(actions, r.randrange(1, kmax + 1)) for _ in range(n - 1)]


def _request(r, kind, roles, actions, scope=None):
    p, res = _attrs(r)
    inp = {"requestId": "u", "actions": list(actions), "principal": {"id": r.choice(["alice", "bob", "carol"]), "roles": list(roles), "attr": p},
           "resource": {"kind": kind, "id": "x", "attr": res}}
    if scope is not None:
        inp["resource"]["scope"] = scope
    return inp


class Case:
    def __init__(self, name, docs, inputs, lenient=False, form=None, staged=True, spec_host=False):
        self.name, self.docs, self.inputs, self.lenient = name, docs, inputs, lenient
        self.form, self.staged, self.spec_host = form, staged, spec_host
        self.rt = build_rule_table(docs)
        self.ft = flatten(self.rt)
        self.enc = Encoder(self.ft.manifest, lenient_scope_search=lenient)
        self.b = self.enc.encode(inputs)
        self.flags = L.BATCH_FLAG_LENIENT if lenient else 0
        self.nR = len(self.ft.manifest["roles"])
        self.n_rows = len(self.enc.row_pat_start)
        self.n_asets = len(np.asarray(self.b.columns[9]))
        rc = self.b.columns[2].shape[0]
        self.rc, self.rcp = rc, 1 << (rc - 1).bit_length()

    @functools.cached_property
    def want(self):
        # raises if oracle #2 flags a request (a run-time value outside the device's exact range): these cases have none
        return cref.check(self.ft.blob, self.b.columns, self.b.n, self.b.max_actions, 0, self.flags, n_threads=os.cpu_count() or 1)

    @functools.cached_property
    def b3(self):
        """the requests three times over: more than two chunks of CHUNK requests each on the host-buffer path"""
        return self.enc.encode(self.inputs * 3)

    @functools.cached_property
    def want3(self):
        return cref.check(self.ft.blob, self.b3.columns, self.b3.n, self.b3.max_actions, 0, self.flags, n_threads=os.cpu_count() or 1)


def _kinds_table(kinds, roles, actions, conds, r, any_role_every=4, drs=None, deny_every=3):
    """policies for `kinds` (one per kind, a different number of rules each): every rule covers a few actions and roles (role
    `*` on every `any_role_every`-th rule, derived roles on every fifth where there are some) and takes the next condition of
    `conds`; every `deny_every`-th rule is a DENY"""
    docs = []
    if drs:
        docs.append({"apiVersion": API, "derivedRoles": {"name": "drs", "definitions": drs}})
    ci = 0
    for k, kind in enumerate(kinds):
        rules = []
        for i in range(3 + (k * 5) % 11):
            acts = r.sample(actions, r.randrange(1, min(4, len(actions)) + 1))
            eff = "D" if i % deny_every == deny_every - 1 else "A"
            if drs and i % 5 == 1:
                rules.append(_rule(acts, eff, derived=[r.choice(drs)["name"]], expr=conds[ci % len(conds)]))
            else:
                rl = ["*"] if i % any_role_every == 0 else r.sample(roles, r.randrange(1, min(3, len(roles)) + 1))
                rules.append(_rule(acts, eff, roles=rl, expr=conds[ci % len(conds)] if i % 4 != 3 else None))
            ci += 1
        docs.append(_rp(kind, rules, drs=bool(drs)))
    return docs


def case_rc1():
    r = random.Random(11)
    actions = [f"a{i}" for i in range(32)]
    kinds = ["k0", "k1", "k2", "k3"]
    docs = _kinds_table(kinds, ["user", "manager", "admin"], actions, _flat_conds(20), r)
    asets = [actions, actions[::-1], actions[:1], actions[3:19], actions[::2], actions[5:]]
    inputs = [_request(r, r.choice(kinds), [r.choice(["user", "manager", "admin", "ghost"])], asets[i % len(asets)]) for i in range(4099)]
    return Case("rc1", docs, inputs, form="mask32", spec_host=True)


def _roles_table(nroles, nkinds, nconds, r, salt):
    roles = [f"r{i}" for i in range(nroles)]
    kinds = [f"k{i}" for i in range(nkinds)]
    return roles, kinds, _kinds_table(kinds, roles, [f"a{i}" for i in range(8)], _flat_conds(nconds, salt), r)


def _roles_inputs(r, roles, kinds, rc, kmax, n):
    out = []
    asets = _asets(r, [f"a{j}" for j in range(8)], kmax)
    for i in range(n):
        nrole = rc if i % 5 == 0 else r.randrange(1, rc + 1)
        rl = r.sample(roles + ["ghost", "nobody"], nrole)
        out.append(_request(r, r.choice(kinds), rl, r.choice(asets)))
    return out


def case_rc5_rw64():
    r = random.Random(12)
    roles, kinds, docs = _roles_table(7, 5, 40, r, 1)
    return Case("rc5_rw64", docs, _roles_inputs(r, roles, kinds, 5, 6, 3001), form="mask64")


def case_rc8():
    r = random.Random(13)
    roles, kinds, docs = _roles_table(7, 5, 40, r, 2)
    return Case("rc8", docs, _roles_inputs(r, roles, kinds, 8, 4, 3001), form="mask64", spec_host=True)


def case_rc4_rw64():
    r = random.Random(14)
    roles, kinds, docs = _roles_table(12, 6, 24, r, 3)
    return Case("rc4_rw64", docs, _roles_inputs(r, roles, kinds, 4, 8, 3001), form="mask32")


def case_index_flat():
    r = random.Random(15)
    conds = _flat_conds(90, 4)
    drs = [{"name": f"dr{i}", "parentRoles": ["user", "manager"][: 1 + i % 2], "condition": {"match": {"expr": conds[(7 * i + 3) % 90]}}} for i in range(5)]
    kinds = [f"k{i}" for i in range(14)]
    docs = _kinds_table(kinds, ["user", "manager", "admin"], [f"a{i}" for i in range(8)], conds, r, drs=drs)
    asets = _asets(r, [f"a{j}" for j in range(8)], 8)
    inputs = [_request(r, r.choice(kinds), r.sample(["user", "manager", "admin", "ghost"], r.randrange(1, 4)), r.choice(asets)) for _ in range(3003)]
    return Case("index_flat", docs, inputs, form="index", spec_host=True)


# scope chains: depth 1-4, REQUIRE_PARENTAL_CONSENT at the root (img), in the middle (doc: a) and at a leaf (doc: a.b.c);
# scope a.b.c holds doc policies but no img policy, scope x only vid policies
CHAIN_SCOPES = {"doc": ["", "a", "a.b", "a.b.c"], "img": ["", "a", "a.b"], "vid": ["", "x"]}
CHAIN_CONSENT = {("doc", "a"), ("doc", "a.b.c"), ("img", "")}


def _chain_docs(r):
    docs = []
    conds = _flat_conds(12, 5)
    for kind, scopes in CHAIN_SCOPES.items():
        for d, sc in enumerate(scopes):
            rules = []
            for i in range(2 + (d + len(kind)) % 3):
                acts = r.sample([f"a{j}" for j in range(6)], r.randrange(1, 4))
                roles = ["*"] if i == 0 else r.sample(["user", "manager", "admin"], 2)
                rules.append(_rule(acts, "A", roles=roles, expr=conds[(3 * d + i) % 12] if i % 2 == 0 else None))
                rules.append(_rule(r.sample([f"a{j}" for j in range(6)], 1), "D", roles=roles, expr=conds[(3 * d + i + 5) % 12]))
            docs.append(_rp(kind, rules, scope=sc, consent=(kind, sc) in CHAIN_CONSENT))
    return docs


def _chain_inputs(r, scopes, n):
    asets = _asets(r, [f"a{j}" for j in range(6)], 6)
    return [_request(r, r.choice(list(CHAIN_SCOPES)), r.sample(["user", "manager", "admin"], r.randrange(1, 3)), r.choice(asets),
                     scope=r.choice(scopes)) for _ in range(n)]


def case_chains():
    r = random.Random(16)
    return Case("chains", _chain_docs(r), _chain_inputs(r, ["", "a", "a.b", "a.b.c", "x", "a.b.c", "a.b"], 3005), form="mask32")


def case_lenient():
    r = random.Random(16)
    docs = _chain_docs(r)
    # exact, deeper than any policy, unknown, and present in the table but not for this kind (img / vid at a.b.c, doc at x)
    return Case("lenient", docs, _chain_inputs(r, ["", "a", "a.b.c", "a.b.c.d.e", "a.b.q", "x.y", "zzz", "x", "a.b"], 3005), lenient=True, form="mask32")


LIST_EXPRS = ["P.attr.dept in R.attr.allowed", "hasIntersection(P.attr.groups, R.attr.allowed)",
              "hasIntersection(R.attr.allowed, P.attr.groups)", "isSubset(R.attr.allowed, P.attr.groups)"]


def _list_value(r, i, lane, numbers):
    """lengths 0..10, absent / null / string / number operands, number elements, strings the table does not hold"""
    k = (lane * 7 + i) % 16
    if k == 0:
        return "absent"
    if k == 1:
        return None
    if k == 2:
        return "g1"
    if k == 3 and numbers:
        return 3
    n = (lane * 3 + i // 32) % 11
    pool = ["g0", "g1", "g2", "g3", "d1"]
    out = [r.choice(pool) if r.random() < 0.6 else f"s{i}_{j}" for j in range(n)]   # s...: batch-only strings
    if numbers and n and r.random() < 0.15:
        out[r.randrange(n)] = r.choice([1, 2.5])
    return out


def _list_inputs(r, n, numbers=True):
    inputs = []
    for i in range(n):
        lane = i % 32
        inp = _request(r, f"k{r.randrange(10)}", ["user"], ["a0", "a1", "a2", "a3", "a4"])
        for msg, key in (("principal", "groups"), ("resource", "allowed")):
            v = _list_value(r, i + (key == "allowed") * 5, lane, numbers)
            if v == "absent":
                inp[msg]["attr"].pop(key, None)
            else:
                inp[msg]["attr"][key] = v
        inp["principal"]["attr"]["dept"] = r.choice(["g1", "g2", "d1", f"s{i}_0", 4, None])
        inputs.append(inp)
    last = inputs[-1]   # the last request's list ends the batch heap; its warp holds longer lists
    last["principal"]["attr"]["groups"] = ["g2"]
    last["resource"]["attr"]["allowed"] = ["g1"]
    return inputs


def _list_docs():
    docs = []
    for k in range(10):   # more block shapes than the block-shape specialiser takes: the table gets the unique-condition one
        rules = [_rule([f"a{j}"], "A", roles=["user"], expr=e) for j, e in enumerate(LIST_EXPRS)]
        rules += [_rule(["a4"], "A", roles=["*"], expr='"g1" in P.attr.groups'), _rule(["a0", "a4"], "D", roles=["user"], expr=f'R.attr.size > {5 + k}')]
        docs.append(_rp(f"k{k}", rules[: 4 + k % 3] + rules[5:]))
    return docs


def case_lists_warp():
    r = random.Random(17)
    return Case("lists_warp", _list_docs(), _list_inputs(r, 32 * 170 + 11), form="mask32", spec_host=True)


def case_global_nopk():
    r = random.Random(18)
    kinds = [f"k{i}" for i in range(90)]
    actions = [f"a{i}" for i in range(8)]
    conds = _flat_conds(30, 6)
    docs = []
    for k, kind in enumerate(kinds):
        rules = [_rule(r.sample(actions, 2), "D" if i % 4 == 3 else "A", roles=[r.choice(["user", "manager", "*"])], expr=conds[(k + i) % 30] if i % 3 else None)
                 for i in range(40 + k % 7)]
        docs.append(_rp(kind, rules))
    inputs = [_request(r, r.choice(kinds), r.sample(["user", "manager", "ghost"], r.randrange(1, 3)), r.sample(actions, r.randrange(1, 9))) for _ in range(4101)]
    return Case("global_nopk", docs, inputs, form="mask32", staged=False)


CASES = {f.__name__[5:]: f for f in (case_rc1, case_rc5_rw64, case_rc8, case_rc4_rw64, case_index_flat, case_chains, case_lenient,
                                     case_lists_warp, case_global_nopk)}


@functools.lru_cache(maxsize=None)
def _case(name):
    return CASES[name]()


# ---- what each case must reach -------------------------------------------------------------------------------------------
def _proves_path(c, src, nu):
    form = next(v for k, v in FORMS.items() if f"kForm = {k}" in src)
    assert form == c.form, (c.name, form, nu)
    assert "kPrograms = false" in src
    rw64 = (c.nR + 1) * c.rcp > 32
    pk = c.n_asets * c.n_rows
    if c.name == "rc1":
        assert c.rc == 1 and c.b.max_actions == 32 and c.b.max_actions * c.rc >= 32
    elif c.name == "rc5_rw64":
        assert c.rc == 5 and c.nR == 7 and (c.nR + 1) * c.rcp == 64 and rw64
    elif c.name == "rc8":
        assert c.rc == 8 and rw64
    elif c.name == "rc4_rw64":
        assert c.rc == 4 and c.nR >= 12 and rw64
        assert any(r.get("roles") == ["*"] for d in c.docs for r in d["resourcePolicy"]["rules"])
    elif c.name == "index_flat":
        assert 64 <= nu <= 127
    elif c.name in ("chains", "lenient"):
        sc = c.enc.scope_ids
        hdr0 = np.asarray(c.b.columns[0]).reshape(-1, 4)
        kinds = [inp["resource"]["kind"] for inp in c.inputs]
        scopes = [inp["resource"].get("scope", "") for inp in c.inputs]
        # chains through a scope that holds no policy for the request's kind (an empty descriptor) ...
        assert sum(s in sc and s not in CHAIN_SCOPES[k] for k, s in zip(kinds, scopes)) >= 200
        # ... and through consent scopes, whose ALLOW rows the descriptors drop
        assert sum(any((k, ".".join(s.split(".")[:j]) if j else "") in CHAIN_CONSENT for j in range(len(s.split(".")) + 1))
                   for k, s in zip(kinds, scopes)) >= 500
        inexact = ((hdr0[:, 2] & L.SCOPE_INEXACT_BIT) != 0) & (hdr0[:, 2] != L.SCOPE_NONE)
        if c.lenient:
            assert inexact.sum() >= 500
        else:
            assert not inexact.any()
    elif c.name == "global_nopk":
        assert pk > 1 << 19 and c.n_asets > 130, (c.n_asets, c.n_rows)
    if c.name != "global_nopk":
        assert pk * 16 < 60 * 1024, (c.name, pk)    # merged rows stay well inside the shared-memory budget


def _list_lengths(c):
    """per request: the list length each list slot of the lists_warp case holds (-1: not a list)"""
    out = []
    for inp in c.inputs:
        out.append([len(v) if isinstance(v, list) else -1 for v in (inp["principal"]["attr"].get("groups"), inp["resource"]["attr"].get("allowed"))])
    return np.array(out)


def _expected_list_deferrals(c):
    """requests the register-list form of the generated evaluator cannot decide: a list longer than 8 or with a non-string
    element where a predicate needs its elements, or a non-list right operand of `in`"""
    n = 0
    for inp in c.inputs:
        a, b, x = inp["principal"]["attr"].get("groups", "absent"), inp["resource"]["attr"].get("allowed", "absent"), inp["principal"]["attr"]["dept"]

        def st(v):   # cb_core.h ListRegs::st
            if v == "absent":
                return 1
            if not isinstance(v, list):
                return 3
            return 2 if len(v) > 8 or any(not isinstance(e, str) for e in v) else 0
        sa, sb = st(a), st(b)
        slow = sb in (2, 3)     # x in B (x is never absent here)
        slow |= sa not in (1, 3) and sb not in (1, 3) and 2 in (sa, sb)
        n += slow
    return n


def _check_shares(c, want):
    valid = want != 0
    allow, deny = (want[valid] == 1).mean(), (want[valid] == 2).mean()
    assert allow >= 0.1 and deny >= 0.1, (c.name, allow, deny)


def _check_oracle1(c, want, k=200):
    orc = CheckOracle(c.rt, lenient_scope_search=c.lenient)
    for j in random.Random(5).sample(range(c.b.n), k):
        got = orc.check(c.inputs[j])["actions"]
        for q, a in enumerate(c.inputs[j]["actions"]):
            assert got[a]["effect"] == want[j, q], (c.name, j, a)


@pytest.mark.parametrize("name", list(CASES))
def test_unique_condition_shapes_host(name, tmp_path):
    """Generated form of each case, oracle #1 vs oracle #2, and the host build of the unique-condition body
    (modes 4 / 5: rows from the image / merged records; generated evaluator once per condition form)."""
    c = _case(name)
    src, nu = hostsim.generate_uc(c.ft.blob)
    assert src, name
    assert hostsim.generate(c.ft.blob) == ""   # too many block shapes for the block-shape specialiser: NVRTC builds this form
    _proves_path(c, src, nu)
    assert c.b.n % 32 != 0 and c.b3.n > 2 * CHUNK and c.b3.n % CHUNK != 0   # ragged warps; the host-buffer path on the device splits
    want = c.want
    _check_shares(c, want)
    _check_oracle1(c, want)
    valid = want != 0      # (padding slots of requests with fewer actions decode as DENY here)
    for mode in (4, 5):
        got = hostsim.check(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body() == mode, (name, mode)   # the table and batch take the unique-condition body
        assert (got[valid] == want[valid]).all(), (name, mode)
    if c.spec_host:
        lib = hostsim.build_spec(c.ft.blob, str(tmp_path), uc=True)
        for mode in (4, 5):
            got = hostsim.check_spec(lib, c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
            assert hostsim.body(lib) == mode, (name, mode)
            assert (got[valid] == want[valid]).all(), (name, mode)
        if name == "lists_warp":
            # the host build bounds each list by its own length: what it defers is exactly the lists the registers cannot hold
            assert hostsim.deferred(lib) == _expected_list_deferrals(c) > c.b.n // 20
            lens = np.minimum(np.maximum(_list_lengths(c), 0), 8)
            n_full = c.b.n // 32 * 32
            w = lens[:n_full].reshape(-1, 32, 2)
            assert ((w.max(axis=1) > w.min(axis=1)).any(axis=1)).sum() >= 100   # warps whose bound exceeds some lane's length
            assert _list_lengths(c).max() == 10 and (_list_lengths(c) == 0).any()
            _assert_heap_ends_with_last_list(c)
            _narrow_batch(c)


# ---- the device ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_unique_condition_shapes_gpu(name, monkeypatch, tmp_path):
    """Each case through the NVRTC-specialised kernel, the ahead-of-time kernel where the image allows it (mask-form rows, no
    programs), and the global-memory image where the staged one fits; device-resident batch and host-buffer path in several
    chunks, against oracle #2."""
    from cerbos_b200 import capi
    from cerbos_b200.device import DeviceBatch
    c = _case(name)
    want = c.want
    assert c.b.n % 32 != 0
    monkeypatch.setenv("CERBOS_B200_UC", "1")
    envs = [{}]
    if c.form != "index":
        envs.append({"CERBOS_B200_NO_JIT": "1"})
    if c.staged:
        envs.append({"CERBOS_B200_NO_STAGE": "1"})
    for env in envs:
        for k in ("CERBOS_B200_NO_JIT", "CERBOS_B200_NO_STAGE", "CERBOS_B200_CHECK_CHUNK"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = capi.Context(0)
        try:
            t = ctx.load_table(c.ft.blob)
            specialised, note = t.wait_ready()
            assert specialised == ("CERBOS_B200_NO_JIT" not in env), (name, env, note)
            d0 = ctx.deferred_count()
            db = DeviceBatch(c.b, "cuda:0")
            db.run(t, 0, c.flags)
            ctx.sync()
            cfg = ctx.last_kernel_config()
            assert cfg["unique_conditions"] and cfg["table_specialised"] == specialised, (name, env, cfg)
            assert (cfg["smem_bytes"] > 0) == (c.staged and "CERBOS_B200_NO_STAGE" not in env), (name, env, cfg)
            got = np.where(want != 0, db.effects(), 0)   # the bitmap has no padding state
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, (name, env, bad[:8].tolist(), got[bad[:4]].tolist(), want[bad[:4]].tolist())
            if name == "lists_warp" and specialised:
                # the warp-wide list bound loads more elements than a lane's own list holds, never fewer: the device defers
                # exactly the requests the host build defers
                lib = hostsim.build_spec(c.ft.blob, str(tmp_path), uc=True)
                hostsim.check_spec(lib, c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=5)
                assert ctx.deferred_count() - d0 == hostsim.deferred(lib), name
            # host-buffer path in chunks of CHUNK requests (the smallest chunk the library takes), the last one partial
            monkeypatch.setenv("CERBOS_B200_CHECK_CHUNK", str(CHUNK))
            assert c.b3.n > 2 * CHUNK and c.b3.n % CHUNK != 0
            host = t.check(c.b3.columns, c.b3.n, c.b3.max_actions, 0, c.flags)
            assert ctx.last_kernel_config()["unique_conditions"]
            assert (host == c.want3).all(), (name, env)
            assert (c.want3[: c.b.n] == want).all()
            if name == "lists_warp" and not env:
                _narrow_run(c, t)
            t.release()
        finally:
            ctx.close()


def _assert_heap_ends_with_last_list(c):
    """the room clamp of cb::list_load: the last request's last list ends the batch heap, and a lane of its (partial) warp holds
    a longer list, so the warp bound asks for words past the end of the heap"""
    slots, heap = np.asarray(c.b.columns[3]), np.asarray(c.b.columns[4])
    tag_list = (L.V64_BOX_BASE | L.V64_LIST)

    def lists(vals):   # heap offsets of the batch lists among `vals`
        return [int(v) & (L.V64_HEAP_BATCH_BIT - 1) for v in vals.ravel() if int(v) >> 48 == tag_list and int(v) & L.V64_HEAP_BATCH_BIT]
    off = max(lists(slots[:, -1]))
    assert off + 1 + int(heap[off]) == len(heap)
    w0 = (c.b.n - 1) // 32 * 32
    assert max(int(heap[o]) for o in lists(slots[:, w0:])) > int(heap[off])


def _narrow_batch(c):
    from cerbos_b200 import narrow as NW
    b = c.enc.encode(_list_inputs(random.Random(19), 32 * 180 + 5, numbers=False))
    nb = NW.narrow_batch(b, len(c.enc.slots))
    assert nb is not None and nb.heap_bits == 16 and nb.heap_base2 >= nb.heap_base + (1 << 14), (nb and nb.heap_bits)
    return b, nb


def _narrow_run(c, t):
    """lists_warp in the narrow wire form: strings only in the lists (numbers keep the heap at 64 bits), so that the heap
    narrows to 16-bit words and the batch-only strings land in its second window"""
    b, nb = _narrow_batch(c)
    want = cref.check(c.ft.blob, b.columns, b.n, b.max_actions, 0, c.flags, n_threads=os.cpu_count() or 1)
    assert (t.check_narrow(nb, 0, c.flags) == want).all()
