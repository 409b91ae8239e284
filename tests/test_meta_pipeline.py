"""Decision metadata (ActionEffect.Policy / Scope, EffectiveDerivedRoles) through the pipelined check path: cgpu_check_meta
and cgpu_check_narrow_meta on workload batches, across chunk boundaries, over the narrow wire (both forms and the native
encoder's route), on several devices, from concurrent callers, and their errors.  The reference for the device is the
metadata body of the host build (hostsim.check_meta), itself held against oracle #1 here on the workload tables."""
import threading

import numpy as np
import pytest

import workloads as W
from cerbos_b200 import meta as M
from cerbos_b200 import narrow as NW
from hostsim import driver as hostsim
from oracle.celeval import parse_timestamp

NOW = parse_timestamp("2024-01-01T00:00:00Z")
NOW_NS = NOW.ns

_built = {}


def _workload(name):
    """-> (workload, rule table, FlatTable, Encoder), built once per module"""
    if name not in _built:
        w = W.WORKLOADS[name]()
        _built[name] = (w, *W.build(w))
    return _built[name]


def _batch(name, n, start=0):
    w, _, _, enc = _workload(name)
    return W.columns_parallel(w, n, start, enc)


def _same_planes(a, b, what):
    for x, y, plane in zip(a, b, ("effects", "action words", "request records")):
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), (what, plane)


# ---- CPU: the metadata body of the host build against oracle #1 on the workload tables ------------------------------------
@pytest.mark.parametrize("name,n", [("C2", 300), ("C3", 300), ("C5", 200)])
def test_host_metadata_body_against_oracle_on_workloads(name, n):
    from oracle.check import CheckOracle
    w, rt, ft, enc = _workload(name)
    f = w.fields(n, start=4321)
    inputs = w.inputs(f, range(n))
    b = enc.encode(inputs)
    eff, am, rm = hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, NOW_NS)
    assert (eff == hostsim.check(ft.blob, b.columns, b.n, b.max_actions, NOW_NS)).all()
    orc = CheckOracle(rt)
    n_pol = 0
    for j, inp in enumerate(inputs):
        py = orc.check(inp, NOW)
        p, r = inp["principal"], inp["resource"]
        for k, a in enumerate(inp["actions"]):
            pol, sc = M.decode_action(int(am[j, k]), rm[j], ft.manifest, p.get("id", ""), r.get("kind", ""),
                                      p.get("policyVersion") or "default", r.get("policyVersion") or "default")
            want = py["actions"][a]
            assert (int(eff[j, k]), pol, sc) == (want["effect"], want["policy"], want["scope"]), (name, j, a)
            n_pol += pol != M.NO_POLICY_MATCH
        assert M.decode_edr(int(rm[j]["effective_derived_roles"]), ft.manifest) == py["effectiveDerivedRoles"], (name, j)
    assert n_pol > 0


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    from cerbos_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def tables(ctx):
    loaded = {}

    def get(name):
        if name not in loaded:
            loaded[name] = ctx.load_table(_workload(name)[2].blob)
        return loaded[name]
    yield get
    for t in loaded.values():
        t.release()


def _meta(t, b):
    return t.check_meta(b.columns, b.n, b.max_actions, NOW_NS)


def _n_slots(name):
    return len(_workload(name)[3].slots)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C2", "C3", "C5"])
def test_meta_at_scale(tables, name):
    """2^20 requests: the effect bytes of cgpu_check_meta equal cgpu_check's.  2^16 requests: its action words and request
    records equal the host build's metadata body over the same columns."""
    t = tables(name)
    ft = _workload(name)[2]
    b = _batch(name, 1 << 20)
    eff, am, rm = _meta(t, b)
    assert (eff == t.check(b.columns, b.n, b.max_actions, NOW_NS)).all(), name
    assert set(np.unique(eff)) <= {1, 2}
    b = _batch(name, 1 << 16, start=1 << 20)
    got = _meta(t, b)
    _same_planes(got, hostsim.check_meta(ft.blob, b.columns, b.n, b.max_actions, NOW_NS), name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C3", "C5"])
def test_meta_across_chunk_boundaries(tables, name, monkeypatch):
    """Chunks of 4096 requests with a ragged last chunk give the same three planes as one chunk, wide and narrow."""
    t = tables(name)
    b = _batch(name, 3 * 4096 + 77)
    nb = NW.narrow_batch(b, _n_slots(name))
    assert nb is not None
    one = (_meta(t, b), t.check_narrow_meta(nb, NOW_NS))
    monkeypatch.setenv("CERBOS_B200_CHECK_CHUNK", "4096")
    chunked = (_meta(t, b), t.check_narrow_meta(nb, NOW_NS))
    _same_planes(chunked[0], one[0], (name, "wide"))
    _same_planes(chunked[1], one[1], (name, "narrow"))
    _same_planes(one[1], one[0], (name, "narrow vs wide"))


@pytest.mark.gpu
@pytest.mark.parametrize("v2", [False, True])
@pytest.mark.parametrize("name,n", [("C2", 50000), ("C3", 50000), ("C5", 20000)])
def test_narrow_meta_equals_wide_meta(tables, name, n, v2):
    t = tables(name)
    b = _batch(name, n, start=777)
    nb = NW.narrow_batch(b, _n_slots(name), v2=v2)
    assert nb is not None
    _same_planes(t.check_narrow_meta(nb, NOW_NS), _meta(t, b), (name, v2))


@pytest.mark.gpu
@pytest.mark.parametrize("lenient", [False, True])
def test_native_route_on_engine_goldens(ctx, lenient):
    """cgpu_encode -> cgpu_narrow_build -> cgpu_check_narrow_meta on the wire messages of the engine goldens: byte-identical to
    cgpu_check_meta on the encoded columns, and the decoded policy / scope / effectiveDerivedRoles are the reference's."""
    from cerbos_b200 import capi, wire
    from cerbos_b200.table.flatten import flatten
    from helpers import engine_decisions, store_rule_table
    names = {"EFFECT_ALLOW": 1, "EFFECT_DENY": 2}
    ft = flatten(store_rule_table(), globals_={"environment": "test"})
    cases = [(cid, inp, want) for cid, len_, inp, want in engine_decisions() if len_ == lenient]
    t = ctx.load_table(ft.blob)
    ne = capi.NativeEncoder(ft.blob, lenient_scope_search=lenient)
    eb = ne.encode([wire.check_input(inp) for _, inp, _ in cases])
    b = eb.batch(NOW_NS)
    wide = t.check_meta(eb.columns(), b.n_requests, b.max_actions, NOW_NS, b.flags)
    n = n_edr = 0
    for form in (1, 2):
        nz = eb.narrow(form)
        assert nz is not None, form
        eff, am, rm = got = t.check_narrow_meta(nz, NOW_NS)
        nz.free()
        _same_planes(got, wide, (lenient, form))
        for j, (cid, inp, want) in enumerate(cases):
            p, r = inp.get("principal") or {}, inp.get("resource") or {}
            for k, a in enumerate(inp["actions"]):
                pol, sc = M.decode_action(int(am[j, k]), rm[j], ft.manifest, p.get("id", ""), r.get("kind", ""),
                                          p.get("policyVersion") or "default", r.get("policyVersion") or "default")
                wa = want["actions"][a]
                assert (int(eff[j, k]), pol, sc) == (names[wa["effect"]], wa.get("policy", ""), wa.get("scope", "")), (cid, a, form)
                n += 1
            wedr = sorted(want.get("effectiveDerivedRoles", want.get("effective_derived_roles")) or [])
            assert M.decode_edr(int(rm[j]["effective_derived_roles"]), ft.manifest) == wedr, (cid, form)
            n_edr += bool(wedr)
    assert n > 0 and (lenient or n_edr > 0)
    eb.free()
    ne.close()
    t.release()


@pytest.mark.gpu
def test_two_devices_equal_one():
    """A context over two devices shards every host-buffer entry point; each gives what a one-device context gives."""
    import torch
    from cerbos_b200 import capi
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least two GPUs")
    for name, n in (("C3", (1 << 17) + 3), ("C5", (1 << 16) + 999)):
        ft = _workload(name)[2]
        b = _batch(name, n)
        nb = NW.narrow_batch(b, _n_slots(name))
        outs = []
        for devices in (0, [0, 1]):
            c = capi.Context(devices)
            t = c.load_table(ft.blob)
            outs.append((t.check(b.columns, b.n, b.max_actions, NOW_NS), t.check_narrow(nb, NOW_NS), _meta(t, b), t.check_narrow_meta(nb, NOW_NS)))
            t.release()
            c.close()
        (e1, n1, m1, nm1), (e2, n2, m2, nm2) = outs
        assert e1.tobytes() == e2.tobytes() and n1.tobytes() == n2.tobytes(), name
        _same_planes(m2, m1, (name, "cgpu_check_meta"))
        _same_planes(nm2, nm1, (name, "cgpu_check_narrow_meta"))


@pytest.mark.gpu
def test_concurrent_callers(tables):
    """8 host threads call cgpu_check_meta / cgpu_check_narrow_meta on different batches at once, on one context: every
    result equals that batch's serial result."""
    t = tables("C3")
    jobs = []
    for i in range(8):
        b = _batch("C3", 40000 + 1000 * i, start=100000 * i)
        if i % 2:
            nb = NW.narrow_batch(b, _n_slots("C3"), v2=i % 4 == 1)
            assert nb is not None
            jobs.append(lambda nb=nb: t.check_narrow_meta(nb, NOW_NS))
        else:
            jobs.append(lambda b=b: _meta(t, b))
    serial = [f() for f in jobs]
    start = threading.Barrier(len(jobs))
    errors = []

    def run(i):
        try:
            start.wait()
            for _ in range(3):
                _same_planes(jobs[i](), serial[i], i)
        except Exception as e:  # noqa: BLE001 -- reported by the main thread
            errors.append((i, e))
    th = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


@pytest.mark.gpu
def test_errors(ctx, tables):
    """A null metadata pointer is an invalid argument; a request the device cannot evaluate exactly (a timestamp beyond 2262)
    fails the narrow metadata call with CGPU_ERR_UNSUPPORTED, and the next call on the context succeeds."""
    import ctypes
    from cerbos_b200 import capi
    from cerbos_b200.encode import Encoder
    from cerbos_b200.policy.compile import build_rule_table
    from cerbos_b200.table.flatten import flatten
    L = capi.lib()
    t = tables("C3")
    b = _batch("C3", 1000)
    nb = NW.narrow_batch(b, _n_slots("C3"))
    bb, nr, keep = t.prepare_narrow(nb, NOW_NS)
    out = np.empty((b.n, b.max_actions), dtype=np.uint8)
    am = np.empty((b.n, b.max_actions), dtype=np.uint32)
    rm = np.empty(b.n, dtype=M.REQUEST_META_DTYPE)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    assert L.cgpu_check_narrow_meta(ctx._h, t._h, ctypes.byref(bb), ctypes.byref(nr), p(out), None, p(rm)) == capi.ERR_INVALID
    assert L.cgpu_check_narrow_meta(ctx._h, t._h, ctypes.byref(bb), ctypes.byref(nr), p(out), p(am), None) == capi.ERR_INVALID
    assert L.cgpu_check_narrow_meta(ctx._h, t._h, ctypes.byref(bb), None, p(out), p(am), p(rm)) == capi.ERR_INVALID
    cols = [np.ascontiguousarray(c) for c in b.columns]
    wb = capi._Batch(b.n, b.max_actions, NOW_NS, 0, (ctypes.c_void_p * 12)(*[c.ctypes.data for c in cols]),
                     (ctypes.c_size_t * 12)(*[c.nbytes for c in cols]), 12)
    assert L.cgpu_check_meta(ctx._h, t._h, ctypes.byref(wb), p(out), p(am), None) == capi.ERR_INVALID
    assert L.cgpu_check_meta(ctx._h, t._h, ctypes.byref(wb), p(out), None, p(rm)) == capi.ERR_INVALID

    pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "doc", "version": "default", "rules": [
        {"actions": ["a"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": "timestamp(R.attr.ts) > now()"}}}]}}
    ft = flatten(build_rule_table([pol]))
    enc = Encoder(ft.manifest)
    tt = ctx.load_table(ft.blob)

    def batch(ts):
        return enc.encode([{"actions": ["a"], "principal": {"id": "p", "roles": ["r"]}, "resource": {"kind": "doc", "id": str(i), "attr": {"ts": s}}}
                           for i, s in enumerate(ts)])
    bad = NW.narrow_batch(batch(["2030-01-01T00:00:00Z", "9999-12-31T23:59:59Z", "2020-01-01T00:00:00Z"]), len(enc.slots))
    with pytest.raises(capi.CgpuError) as e:
        tt.check_narrow_meta(bad, NOW_NS)
    assert e.value.code == capi.ERR_UNSUPPORTED
    good = NW.narrow_batch(batch(["2030-01-01T00:00:00Z", "2020-01-01T00:00:00Z"]), len(enc.slots))
    eff, _, _ = tt.check_narrow_meta(good, NOW_NS)
    assert eff[:, 0].tolist() == [1, 2]
    assert tt.check_narrow(good, NOW_NS)[:, 0].tolist() == [1, 2]
    tt.release()
    del keep
