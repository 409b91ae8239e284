"""The segment form of the unique-condition image (cb_uc.h): every policy block gets the same number of DENY slots followed
by the same number of ALLOW slots, each the largest over the table's blocks, and the specialised walk (cb::uc_walk) runs
them at constant offsets with no per-row clamp or effect test.  The table here pads unevenly: its most DENY rows and its
most ALLOW rows come from different blocks, one block holds only DENY rows and one only ALLOW rows, some scopes ask for
parental consent (their ALLOW mask is zero; one holds more DENY rows than the DENY slots, which then fill its ALLOW slots
too), some requests name a scope without a block for their kind (the empty segment
0), and the batch has several action sets.  Host build of the generic and the generated body, the device kernels, oracle
#2 on every request and oracle #1 on a sample."""
import os
import random
import sys

import numpy as np
import pytest

from hostsim import driver as hostsim
from test_uc_shapes import Case, _asets, _check_oracle1, _check_shares, _flat_conds, _request, _rp, _rule

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from uc_walk_steps import walk_rows  # noqa: E402

ACTIONS = [f"a{j}" for j in range(6)]
# kind -> (DENY rules, ALLOW rules) of its policy in every scope it has one
SHAPES = {"deny_heavy": (5, 1), "allow_heavy": (1, 6), "deny_only": (3, 0), "allow_only": (0, 4), "mixed": (2, 2)}
SCOPES = ["", "a", "a.b"]
CONSENT = {"a"}


def _segment_docs(r):
    conds = _flat_conds(18, 3)
    docs = []
    for k, (kind, (n_deny, n_allow)) in enumerate(SHAPES.items()):
        for d, sc in enumerate(SCOPES):
            if kind == "mixed" and sc == "a.b":
                continue   # a scope without a block for this kind
            rules = []
            # in the consent scope, more DENY rows than any block whose ALLOWs count: they fill the ALLOW slots too
            for i in range(n_deny + 3 * (kind == "deny_heavy" and sc in CONSENT)):
                rules.append(_rule(r.sample(ACTIONS, r.randrange(1, 4)), "D", roles=[r.choice(["user", "manager", "*"])], expr=conds[(k + 5 * d + i) % 18]))
            for i in range(n_allow):
                rules.append(_rule(r.sample(ACTIONS, r.randrange(1, 4)), "A", roles=[r.choice(["user", "manager", "*"])],
                                   expr=conds[(2 * k + d + i + 7) % 18] if i % 3 != 2 else None))
            docs.append(_rp(kind, rules, scope=sc, consent=sc in CONSENT))
    return docs


def _case():
    r = random.Random(31)
    asets = _asets(r, ACTIONS, 6)
    inputs = [_request(r, r.choice(list(SHAPES)), r.sample(["user", "manager", "admin", "ghost"], r.randrange(1, 4)), r.choice(asets),
                       scope=r.choice(SCOPES)) for _ in range(4005)]
    return Case("segments", _segment_docs(r), inputs, spec_host=True)


_cached = []


def _c():
    if not _cached:
        _cached.append(_case())
    return _cached[0]


def _slots(src):
    return [int(src.split(f"{k} = ")[1].split("u")[0]) for k in ("kDenyRows", "kAllowRows", "kScopeRows")]


def test_segment_layout():
    """the generated walk takes the segment form, and the table pads unevenly, as its docstring says"""
    c = _c()
    src, _ = hostsim.generate_uc(c.ft.blob)
    assert src and hostsim.generate(c.ft.blob) == ""
    n_deny, n_allow, scope_rows = _slots(src)
    assert n_deny == 5 and n_allow == 6 and scope_rows == n_deny + n_allow, (n_deny, n_allow, scope_rows)
    assert c.n_asets > 1
    rows, walked = walk_rows(c.ft.blob, c.b, c.flags)
    assert walked == scope_rows
    lv = rows.reshape(-1, 2).astype(int)
    lv = lv[lv.sum(axis=1) > 0]
    assert ((lv[:, 0] == n_deny) & (lv[:, 1] < n_allow)).any()        # the most DENY rows: a block with few ALLOW rows
    assert ((lv[:, 1] == n_allow) & (lv[:, 0] < n_deny)).any()        # the most ALLOW rows: another block
    assert ((lv[:, 0] == 0) & (lv[:, 1] > 0)).sum() > 100             # ALLOW-only blocks
    assert ((lv[:, 0] > 0) & (lv[:, 1] == 0)).sum() > 300             # DENY-only blocks and consent scopes
    assert ((lv[:, 0] > n_deny) & (lv[:, 1] == 0)).sum() > 50         # DENY rows in the ALLOW slots
    kinds = [inp["resource"]["kind"] for inp in c.inputs]
    scopes = [inp["resource"]["scope"] for inp in c.inputs]
    assert sum(k == "mixed" and s == "a.b" for k, s in zip(kinds, scopes)) > 200   # chains through the empty segment
    assert sum(s.startswith("a") for s in scopes) > 1000                                  # chains through the consent scope


def test_segments_host(tmp_path):
    c = _c()
    want = c.want
    _check_shares(c, want)
    _check_oracle1(c, want)
    valid = want != 0
    for mode in (4, 5):
        got = hostsim.check(c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body() == mode
        assert (got[valid] == want[valid]).all(), mode
    lib = hostsim.build_spec(c.ft.blob, str(tmp_path), uc=True)
    for mode in (4, 5):
        got = hostsim.check_spec(lib, c.ft.blob, c.b.columns, c.b.n, c.b.max_actions, 0, c.flags, mode=mode)
        assert hostsim.body(lib) == mode
        assert (got[valid] == want[valid]).all(), mode


@pytest.mark.gpu
def test_segments_gpu(monkeypatch):
    """through the NVRTC-specialised kernel, the ahead-of-time one and the global-memory image (merged-row pre-pass), against
    oracle #2"""
    from cerbos_b200 import capi
    from cerbos_b200.device import DeviceBatch
    c = _c()
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
            assert specialised == ("CERBOS_B200_NO_JIT" not in env), (env, note)
            db = DeviceBatch(c.b, "cuda:0")
            db.run(t, 0, c.flags)
            ctx.sync()
            cfg = ctx.last_kernel_config()
            assert cfg["unique_conditions"] and cfg["table_specialised"] == specialised, (env, cfg)
            assert (cfg["smem_bytes"] > 0) == ("CERBOS_B200_NO_STAGE" not in env), (env, cfg)
            got = np.where(want != 0, db.effects(), 0)
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, (env, bad[:8].tolist())
            t.release()
        finally:
            ctx.close()
