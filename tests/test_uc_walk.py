"""The unique-condition walk (cb::uc_walk) on scopes whose rows it routes by effect in one pass: DENY and ALLOW rows of one
scope that hit the same (action, role) pair, scopes whose ALLOWs do not count (REQUIRE_PARENTAL_CONSENT), and a table
whose longest scope is past the unroll bound of the specialised walk (kUcUnrollRows), so that the generated evaluator
takes the looping form.  Same checks as test_uc_shapes.py: host build of the generic and the generated body, the device
kernels, oracle #2 on every request and oracle #1 on a sample."""
import os
import random
import sys

import numpy as np
import pytest

from hostsim import driver as hostsim
from test_uc_shapes import Case, _asets, _check_oracle1, _check_shares, _flat_conds, _request, _rp, _rule

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from uc_walk_steps import walk_rows, warp_steps  # noqa: E402

UNROLL_ROWS = 16   # cb_core.h: kUcUnrollRows


def _scope_rows(src):
    return int(src.split("kScopeRows = ")[1].split("u;")[0])


def _same_pair_docs(r, n_pairs, max_roles):
    """per (kind, scope): n_pairs (+ 0..2) rule pairs, an ALLOW and a DENY on the same actions and roles under different
    conditions, plus one unconditional ALLOW; kinds differ in rule count (many block shapes); scope a.b asks for
    parental consent (scope permissions belong to the scope, not to one kind's policy)"""
    conds = _flat_conds(24, 2)
    actions = [f"a{j}" for j in range(6)]
    docs = []
    for k in range(12):
        for d, sc in enumerate(["", "a", "a.b"]):
            rules = []
            for i in range(n_pairs + k % 3):
                acts = r.sample(actions, r.randrange(1, 4))
                roles = ["*"] if i % 4 == 0 else r.sample(["user", "manager", "admin"], r.randrange(1, max_roles + 1))
                rules.append(_rule(acts, "A", roles=roles, expr=conds[(k + 3 * d + i) % 24]))
                rules.append(_rule(acts, "D", roles=roles, expr=conds[(k + 3 * d + i + 7) % 24]))
            rules.append(_rule(r.sample(actions, 2), "A", roles=[r.choice(["user", "manager"])]))
            docs.append(_rp(f"k{k}", rules, scope=sc, consent=sc == "a.b"))
    return docs


def _inputs(r, n):
    asets = _asets(r, [f"a{j}" for j in range(6)], 6)
    return [_request(r, f"k{r.randrange(12)}", r.sample(["user", "manager", "admin", "ghost"], r.randrange(1, 4)), r.choice(asets),
                     scope=r.choice(["", "a", "a.b", "a.b"])) for _ in range(n)]


def case_same_pair():
    r = random.Random(21)
    return Case("same_pair", _same_pair_docs(r, 2, 1), _inputs(r, 4001), spec_host=True)


def case_long_scope():
    r = random.Random(22)
    return Case("long_scope", _same_pair_docs(r, 9, 2), _inputs(r, 4003), spec_host=True)


CASES = {"same_pair": case_same_pair, "long_scope": case_long_scope}
_cache = {}


def _case(name):
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]


@pytest.mark.parametrize("name", list(CASES))
def test_walk_host(name, tmp_path):
    c = _case(name)
    src, _ = hostsim.generate_uc(c.ft.blob)
    assert src and hostsim.generate(c.ft.blob) == ""   # the unique-condition form, not the block-shape one
    rows = _scope_rows(src)
    assert (rows <= UNROLL_ROWS) == (name == "same_pair"), rows
    want = c.want
    _check_shares(c, want)
    _check_oracle1(c, want)
    valid = want != 0
    for mode in (4, 5):
        got = hostsim.check(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body() == mode
        assert (got[valid] == want[valid]).all(), (name, mode)
    lib = hostsim.build_spec(c.ft.blob, str(tmp_path), uc=True)
    for mode in (4, 5):
        got = hostsim.check_spec(lib, c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body(lib) == mode
        assert (got[valid] == want[valid]).all(), (name, mode)


def test_walk_rows_per_scope():
    """the chain descriptors of the same-pair table: DENY and ALLOW rows in one scope, consent scopes without ALLOW rows,
    and a longest scope equal to the generated unroll bound"""
    c = _case("same_pair")
    rows, scope_rows = walk_rows(c.ft.blob, c.b, c.flags)
    assert scope_rows == _scope_rows(hostsim.generate_uc(c.ft.blob)[0])
    lv = rows.reshape(-1, 2)
    assert ((lv[:, 0] > 0) & (lv[:, 1] > 0)).sum() > 1000        # scopes with both kinds of row
    assert ((lv[:, 0] > 0) & (lv[:, 1] == 0)).sum() > 300        # consent scopes: their ALLOW rows do not count
    assert (lv.sum(axis=1) <= scope_rows).all()
    s = warp_steps(rows, scope_rows)
    assert (s["one pass"] <= s["two loops"]).all() and (s["one pass"] <= s["unrolled"]).all()
    assert s["one pass"].sum() < s["two loops"].sum()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_walk_gpu(name, monkeypatch):
    """each case through the NVRTC-specialised kernel, the ahead-of-time one and the global-memory image, against oracle #2"""
    from cerbos_b200 import capi
    from cerbos_b200.device import DeviceBatch
    c = _case(name)
    want = c.want
    monkeypatch.setenv("CERBOS_B200_UC", "1")
    for env in ({}, {"CERBOS_B200_NO_JIT": "1"}, {"CERBOS_B200_NO_STAGE": "1"}):
        for k in ("CERBOS_B200_NO_JIT", "CERBOS_B200_NO_STAGE"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = capi.Context(0)
        try:
            t = ctx.load_table(c.ft.blob)
            specialised, note = t.wait_ready()
            assert specialised == ("CERBOS_B200_NO_JIT" not in env), (name, env, note)
            db = DeviceBatch(c.b, "cuda:0")
            db.run(t, 0, c.flags)
            ctx.sync()
            cfg = ctx.last_kernel_config()
            assert cfg["unique_conditions"] and cfg["table_specialised"] == specialised, (name, env, cfg)
            got = np.where(want != 0, db.effects(), 0)
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, (name, env, bad[:8].tolist())
            t.release()
        finally:
            ctx.close()
