"""GPU parity tests: the CUDA path, called through the C ABI, against the oracles (bit-exact)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NOW_NS = 1_704_067_200_000_000_000  # 2024-01-01T00:00:00Z


@pytest.fixture(scope="module")
def ctx():
    from cerbos_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


def _names(eff):
    return {"EFFECT_ALLOW": 1, "EFFECT_DENY": 2}[eff]


def test_engine_goldens_through_engine_api():
    """166 reference engine goldens through Engine.check (host-buffer C ABI)."""
    from cerbos_b200.engine import Engine
    from helpers import engine_decisions, load_golden
    docs = [e["policy"] for e in load_golden("store_policies.json")]
    engines = {False: Engine(docs, globals_={"environment": "test"}),
               True: Engine(docs, globals_={"environment": "test"}, lenient_scope_search=True)}
    n = 0
    for cid, lenient, inp, want in engine_decisions():
        got = engines[lenient].check([inp], now_ns=NOW_NS)[0]
        assert got["requestId"] == inp.get("requestId", "") and got["resourceId"] == inp["resource"]["id"]
        for a, wv in want["actions"].items():
            assert got["actions"][a]["effect"] == wv["effect"], (cid, a)
            n += 1
    assert n == 166
    for e in engines.values():
        e.close()


def test_goldens_batched_device_vs_oracle(ctx):
    from cerbos_b200.device import DeviceBatch
    from cerbos_b200.encode import Encoder
    from cerbos_b200.table.flatten import flatten
    from helpers import engine_decisions, store_rule_table
    from oracle import cref
    ft = flatten(store_rule_table(), globals_={"environment": "test"})
    table = ctx.load_table(ft.blob)
    inputs = [inp for _, lenient, inp, _ in engine_decisions() if not lenient]
    b = Encoder(ft.manifest).encode(inputs * 40)   # > 1 tile, mixed shapes
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, NOW_NS)
    db = DeviceBatch(b, "cuda:0")
    db.run(table, NOW_NS)
    ctx.sync()
    got = db.effects()
    valid = want != 0
    assert (got[valid] == want[valid]).all()
    host = table.check(b.columns, b.n, b.max_actions, NOW_NS)
    assert (host == want).all()
    table.release()


@pytest.mark.parametrize("name,n", [("C1", 1024), ("C2", 1 << 16), ("C2", 1 << 20), ("C3", 1 << 16), ("C3", 1 << 20)])
def test_workloads_bit_exact(ctx, name, n):
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
    table = ctx.load_table(ft.blob)
    db = DeviceBatch(b, "cuda:0")
    db.run(table)
    ctx.sync()
    got = db.effects()
    assert (got == want).all()
    # size-independent properties: every decision is ALLOW or DENY; re-running is idempotent; checksum of checksums
    assert set(np.unique(got)) <= {1, 2}
    db.run(table)
    ctx.sync()
    assert (db.effects() == got).all()
    host = table.check(b.columns, b.n, b.max_actions)
    assert (host == want).all()
    assert int(host.astype(np.uint64).sum()) == int(want.astype(np.uint64).sum())
    table.release()


def test_staged_and_global_table_paths_agree():
    """The TMA-staged (shared memory) and the global-memory table paths give identical bits."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    w = W.C2()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(1 << 16), enc)
    outs = []
    for flag in ("0", "1"):
        os.environ["CERBOS_B200_NO_STAGE"] = flag
        c = capi.Context(0)
        t = c.load_table(ft.blob)
        db = DeviceBatch(b, "cuda:0")
        db.run(t)
        c.sync()
        outs.append((db.effects(), c.last_kernel_config()))
        t.release()
        c.close()
    os.environ.pop("CERBOS_B200_NO_STAGE", None)
    assert outs[0][1]["smem_bytes"] > 0 and outs[1][1]["smem_bytes"] == 0
    assert (outs[0][0] == outs[1][0]).all()


def test_lean_and_general_kernel_bodies_agree():
    """CERBOS_B200_FORCE_GENERAL=1 disables the lean body: both must give identical bits."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    for name in ("C2", "C3"):
        w = W.WORKLOADS[name]()
        _, ft, enc = W.build(w)
        b = w.columns(w.fields(1 << 15), enc)
        outs = []
        for flag in ("0", "1"):
            os.environ["CERBOS_B200_FORCE_GENERAL"] = flag
            c = capi.Context(0)
            t = c.load_table(ft.blob)
            db = DeviceBatch(b, "cuda:0")
            db.run(t)
            c.sync()
            outs.append((db.effects(), c.last_kernel_config()))
            t.release()
            c.close()
        os.environ.pop("CERBOS_B200_FORCE_GENERAL", None)
        assert outs[0][1]["lean_body"] and not outs[1][1]["lean_body"]
        assert (outs[0][0] == outs[1][0]).all(), name


def test_error_paths(ctx):
    from cerbos_b200 import capi
    import workloads as W
    with pytest.raises(capi.CgpuError):
        ctx.load_table(b"\0" * 64)
    w = W.C1()
    _, ft, enc = W.build(w)
    t = ctx.load_table(ft.blob)
    b = w.columns(w.fields(), enc)
    cols = list(b.columns)
    cols[2] = cols[2][:, :100]   # roles column no longer a multiple of n
    with pytest.raises(capi.CgpuError):
        t.check(cols, b.n, b.max_actions)
    t.release()


def test_many_actions_multiple_passes(ctx):
    import workloads as W
    from cerbos_b200.encode import Encoder
    from cerbos_b200.policy.compile import build_rule_table
    from cerbos_b200.table.flatten import flatten
    from oracle import cref
    rt = build_rule_table(W.C2().policies())
    ft = flatten(rt)
    acts = list(dict.fromkeys([f"a{i % 8}" if i % 3 else f"zz{i}" for i in range(70)]))
    inputs = []
    for j in range(300):
        inputs.append({"actions": acts[: 1 + j % len(acts)],
                       "principal": {"id": f"p{j % 7}", "roles": ["user", "manager", "admin", "x1", "x2"][: 1 + j % 5], "attr": {"dept": f"d{j % 3}"}},
                       "resource": {"kind": f"kind_{j % 10}", "id": "r", "attr": {"owner": f"p{j % 5}", "dept": f"d{j % 2}", "status": ["OPEN", "CLOSED"][j % 2], "locked": j % 11 == 0}}})
    b = Encoder(ft.manifest).encode(inputs)
    assert b.n_pass > 1
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    t = ctx.load_table(ft.blob)
    got = t.check(b.columns, b.n, b.max_actions)
    assert (got == want).all()
    t.release()


@pytest.mark.parametrize("name,n", [("C2", (1 << 16) + 777), ("C3", (1 << 18) + 5), ("C2", 1000)])
def test_clustered_and_index_order_agree(name, n):
    """CERBOS_B200_CLUSTER=1 forces the clustering kernels (requests grouped by policy block), =0 disables them:
    identical bits, host-buffer and device paths, sizes that are not multiples of the chunk / window."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
    for flag in ("0", "1"):
        os.environ["CERBOS_B200_CLUSTER"] = flag
        c = capi.Context(0)
        t = c.load_table(ft.blob)
        db = DeviceBatch(b, "cuda:0")
        db.run(t)
        c.sync()
        cfg = c.last_kernel_config()
        assert cfg["clustered"] == (flag == "1")
        assert (db.effects() == want).all(), (name, flag)
        assert (t.check(b.columns, b.n, b.max_actions) == want).all(), (name, flag, "host")
        t.release()
        c.close()
    os.environ.pop("CERBOS_B200_CLUSTER", None)


def test_clustered_goldens_mixed_shapes():
    """The reference goldens (principal / role policies, globs: general body) evaluated in clustered order."""
    from cerbos_b200 import capi
    from cerbos_b200.encode import Encoder
    from cerbos_b200.table.flatten import flatten
    from helpers import engine_decisions, store_rule_table
    from oracle import cref
    ft = flatten(store_rule_table(), globals_={"environment": "test"})
    inputs = [inp for _, lenient, inp, _ in engine_decisions() if not lenient]
    b = Encoder(ft.manifest).encode(inputs * 100)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, NOW_NS)
    os.environ["CERBOS_B200_CLUSTER"] = "1"
    c = capi.Context(0)
    t = c.load_table(ft.blob)
    got = t.check(b.columns, b.n, b.max_actions, NOW_NS)
    assert c.last_kernel_config()["clustered"]
    os.environ.pop("CERBOS_B200_CLUSTER", None)
    assert (got == want).all()
    t.release()
    c.close()


@pytest.mark.parametrize("name,n", [("C2", (1 << 16) + 260), ("C2", (1 << 16) + 777), ("C1", 1024), ("C2", 200)])
def test_tma_column_tiles_and_direct_loads_agree(name, n):
    """Index-order lean launches stage the request columns through TMA (double-buffered 256-request tiles) when the
    column runs are 16-byte aligned; CERBOS_B200_NO_TILES=1 forces the per-thread global loads.  Covers a ragged last
    tile, a batch whose stride is not a multiple of 4 (must fall back) and a batch smaller than one tile."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
    used = {}
    for flag in ("0", "1"):
        os.environ["CERBOS_B200_NO_TILES"] = flag
        c = capi.Context(0)
        t = c.load_table(ft.blob)
        db = DeviceBatch(b, "cuda:0")
        db.run(t)
        c.sync()
        used[flag] = c.last_kernel_config()["tma_column_tiles"]
        assert (db.effects() == want).all(), (name, n, flag)
        assert (t.check(b.columns, b.n, b.max_actions) == want).all(), (name, n, flag, "host")
        t.release()
        c.close()
    os.environ.pop("CERBOS_B200_NO_TILES", None)
    assert used["1"] is False
    assert used["0"] == (n % 4 == 0)


@pytest.mark.parametrize("name,n", [("C2", (1 << 16) + 260), ("C2", 4099), ("C1", 1024), ("C3", 1 << 15)])
def test_table_specialised_and_generic_kernels_agree(name, n):
    """The kernels compiled for the table at run time (cb_specialize.h + NVRTC) against the ahead-of-time generic
    ones (CERBOS_B200_NO_JIT=1) and the oracle; tile-staged and direct column paths, clustered and index order."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
    seen = {}
    for nojit in ("0", "1"):
        for cluster in ("0", "1"):
            os.environ["CERBOS_B200_NO_JIT"] = nojit
            os.environ["CERBOS_B200_CLUSTER"] = cluster
            c = capi.Context(0)
            t = c.load_table(ft.blob)
            t.wait_ready()
            db = DeviceBatch(b, "cuda:0")
            db.run(t)
            c.sync()
            cfg = c.last_kernel_config()
            seen[(nojit, cluster)] = cfg
            assert (db.effects() == want).all(), (name, n, nojit, cluster)
            assert (t.check(b.columns, b.n, b.max_actions) == want).all(), (name, n, nojit, cluster, "host")
            t.release()
            c.close()
    os.environ.pop("CERBOS_B200_NO_JIT", None)
    os.environ.pop("CERBOS_B200_CLUSTER", None)
    # C3 (75 block shapes) gets the unique-condition form of the specialised kernels, index order only
    assert seen[("0", "0")]["table_specialised"] and not seen[("1", "0")]["table_specialised"]
    assert seen[("0", "0")]["unique_conditions"] == (name == "C3") and not seen[("0", "1")]["unique_conditions"]


def test_specialised_kernel_defers_to_general_kernel():
    """Requests the lean body cannot decide (principal and resource policy versions differ) travel through the
    deferral list of the specialised kernel to the general kernel."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.C2()
    _, ft, enc = W.build(w)
    f = w.fields(3000)
    inputs = w.inputs(f, range(3000))
    for i in range(0, 3000, 7):
        inputs[i]["principal"]["policyVersion"] = "v2"
    for i in range(3, 3000, 11):
        inputs[i]["resource"]["attr"]["owner"] = ["a", "list"]          # container equality: out of the 8-byte fast forms
    b = enc.encode(inputs)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions)
    for nojit in ("0", "1"):
        os.environ["CERBOS_B200_NO_JIT"] = nojit
        c = capi.Context(0)
        t = c.load_table(ft.blob)
        t.wait_ready()
        db = DeviceBatch(b, "cuda:0")
        db.run(t)
        c.sync()
        assert c.last_kernel_config()["table_specialised"] == (nojit == "0")
        assert (db.effects() == want).all(), nojit
        assert (t.check(b.columns, b.n, b.max_actions) == want).all(), nojit
        t.release()
        c.close()
    os.environ.pop("CERBOS_B200_NO_JIT", None)


def test_workload_c5_adversarial(ctx):
    """BASELINE.json configs[4] (1000 policies, deep CEL, JWT claims, Zipf kinds): 73 distinct conditions, 50 of them
    without a flat form, table image > 96 KB.  Before the specialised kernel is compiled the general body (bytecode
    interpreter) answers; once it is loaded, cb_spec_uc_global -- every leaf program as straight-line code, table read
    through L2 -- decides every request itself.  Both bit-exact against the oracle."""
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.C5()
    _, ft, enc = W.build(w)
    f = w.fields(8192)
    b = enc.encode(w.inputs(f, range(f["n"])))
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, NOW_NS, n_threads=os.cpu_count() or 1)
    os.environ["CERBOS_B200_NO_JIT"] = "1"
    try:
        from cerbos_b200 import capi
        c0 = capi.Context(0)
        t0 = c0.load_table(ft.blob)
        assert t0.wait_ready()[0] is False
        db = DeviceBatch(b, "cuda:0")
        db.run(t0, NOW_NS)
        c0.sync()
        assert (db.effects() == want).all()
        assert c0.last_kernel_config()["unique_conditions"] is False
        t0.release()
        c0.close()
    finally:
        os.environ.pop("CERBOS_B200_NO_JIT", None)
    table = ctx.load_table(ft.blob)
    specialised, note = table.wait_ready()
    assert specialised, note
    db = DeviceBatch(b, "cuda:0")
    db.run(table, NOW_NS)
    ctx.sync()
    cfg = ctx.last_kernel_config()
    assert cfg["unique_conditions"] and cfg["table_specialised"] and cfg["smem_bytes"] == 0, cfg      # too large to stage
    assert (db.effects() == want).all()
    assert (table.check(b.columns, b.n, b.max_actions, NOW_NS) == want).all()
    table.release()


def test_check_resources_api_goldens_through_engine_api():
    """The reference's API-level CheckResources goldens (cr_case_00 ... 08, 48 decisions) through Engine.check on the GPU."""
    from cerbos_b200.engine import Engine
    from helpers import check_resources_api_cases, load_golden
    docs = [e["policy"] for e in load_golden("store_policies.json")]
    eng = Engine(docs, globals_={"environment": "test"})
    n = 0
    for f, ci, want in check_resources_api_cases():
        got = eng.check([ci], now_ns=NOW_NS)[0]
        for a, w in want.items():
            assert got["actions"][a]["effect"] == w, (f, a)
            n += 1
    assert n == 48
    eng.close()


def test_verify_suite_goldens_through_engine_api():
    """145 engine answers recorded by the reference's policy-test goldens (verify/cases) through Engine.check on the GPU, under
    every engine configuration the suites use (globals, default policy version / scope, lenient scope search, now)."""
    import json
    from cerbos_b200.engine import Engine
    from helpers import load_golden, verify_suite_cases
    from oracle.celeval import parse_timestamp
    docs = [e["policy"] for e in load_golden("store_policies.json")]
    n = 0
    for (gl, dver, dscope, lenient), cases in verify_suite_cases():
        eng = Engine(docs, globals_=json.loads(gl), default_policy_version=dver, default_scope=dscope, lenient_scope_search=lenient)
        for c in cases:
            now_ns = parse_timestamp(c["now"]).ns if c["now"] else NOW_NS
            got = eng.check([c["input"]], now_ns=now_ns)[0]
            for a, w in c["want"].items():
                assert got["actions"][a]["effect"] == w, (c["file"], c["test"], a)
                n += 1
        eng.close()
    assert n == 145


@pytest.mark.parametrize("name,n", [("C3", (1 << 18) + 77), ("C2", (1 << 16) + 5)])
def test_unique_condition_kernels(name, n):
    """Unique-condition kernels (cb_uc.h image, cb::eval_request_uc): the ahead-of-time generic form, the NVRTC-specialised
    form, staged and global table paths -- all against the oracle; device path and host-buffer path."""
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = w.columns(w.fields(n), enc)
    want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
    seen = set()
    for env in ({"CERBOS_B200_UC": "1", "CERBOS_B200_NO_JIT": "1"}, {"CERBOS_B200_UC": "1", "CERBOS_B200_NO_JIT": "1", "CERBOS_B200_NO_STAGE": "1"},
                {"CERBOS_B200_UC": "1"}):
        os.environ.update(env)
        try:
            c = capi.Context(0)
            t = c.load_table(ft.blob)
            t.wait_ready()
            db = DeviceBatch(b, "cuda:0")
            db.run(t)
            c.sync()
            cfg = c.last_kernel_config()
            assert cfg["unique_conditions"] and not cfg["clustered"], cfg
            seen.add((cfg["table_specialised"], cfg["smem_bytes"] > 0))
            assert (db.effects() == want).all(), env
            assert (t.check(b.columns, b.n, b.max_actions) == want).all(), env
            t.release()
            c.close()
        finally:
            for k in env:
                os.environ.pop(k, None)
    if name == "C3":
        assert (True, True) in seen and (False, True) in seen and (False, False) in seen, seen


def test_unique_condition_kernel_deferral_list():
    """Requests the unique-condition body cannot decide (differing policy versions) travel through the launch's deferral
    list to the general kernel -- several launches in flight on several streams, each with its own list."""
    import torch
    from cerbos_b200 import capi
    import workloads as W
    from cerbos_b200.device import DeviceBatch
    from oracle import cref
    w = W.C3()
    _, ft, enc = W.build(w)
    n = 1 << 16
    os.environ["CERBOS_B200_UC"] = "1"
    try:
        c = capi.Context(0)
        t = c.load_table(ft.blob)
        t.wait_ready()
        batches, wants = [], []
        for j in range(4):
            b = w.columns(w.fields(n, start=j * n), enc)
            hdr1 = b.columns[1].copy()
            hdr1["pv"][j::7] = 0xFFFF            # no principal policy version: pv != rv -> deferred
            b.columns[1] = hdr1
            wants.append(cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1))
            batches.append(DeviceBatch(b, "cuda:0"))
        streams = [torch.cuda.Stream() for _ in range(4)]
        for rep in range(3):
            for j, db in enumerate(batches):
                db.run(t, stream=streams[(j + rep) % 4].cuda_stream)
        torch.cuda.synchronize()
        for db, want in zip(batches, wants):
            assert (db.effects() == want).all()
        t.release()
        c.close()
    finally:
        os.environ.pop("CERBOS_B200_UC", None)


def test_cgpu_check_is_reentrant_across_threads():
    """16 host threads call cgpu_check concurrently (as gRPC goroutines call engine.Check, cerbos_svc.go:156, 205, 265):
    batches of different sizes, some with requests the lean kernels defer (differing policy versions), pipelined in chunks
    (CERBOS_B200_CHECK_CHUNK small, so every call is multi-chunk).  Every result must match the oracle."""
    import threading
    from cerbos_b200 import capi
    import workloads as W
    from oracle import cref
    os.environ["CERBOS_B200_CHECK_CHUNK"] = "8192"
    try:
        c = capi.Context(0)
        tables, jobs = {}, []
        for name in ("C2", "C3"):
            w = W.WORKLOADS[name]()
            _, ft, enc = W.build(w)
            t = c.load_table(ft.blob)
            t.wait_ready()
            tables[name] = t
            for j in range(8):
                n = 20000 + 4099 * j
                b = w.columns(w.fields(n, start=j * 50000), enc)
                hdr1 = b.columns[1].copy()
                hdr1["pv"][j::11] = 0xFFFF            # pv != rv -> deferred to the general kernel
                b.columns[1] = hdr1
                want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
                jobs.append((name, b, want))
        errors = []

        def run(job):
            name, b, want = job
            try:
                for _ in range(3):
                    got = tables[name].check(b.columns, b.n, b.max_actions)
                    if not (got == want).all():
                        errors.append((name, b.n, int((got != want).sum())))
            except Exception as e:  # noqa: BLE001
                errors.append((name, b.n, repr(e)))

        threads = [threading.Thread(target=run, args=(j,)) for j in jobs]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errors, errors
        for t in tables.values():
            t.release()
        c.close()
    finally:
        os.environ.pop("CERBOS_B200_CHECK_CHUNK", None)


def test_run_time_values_on_gpu():
    """The list / string producing functions, collecting comprehensions, dynamic literals and hierarchy(list) on the
    device (per-thread scratch arena of the general kernel) against oracle #1 -- same cases as the CPU test of the
    kernel core -- plus every golden CEL leaf that builds values at run time."""
    from cerbos_b200.encode import Encoder
    from oracle.check import CheckOracle
    from oracle.celeval import parse_timestamp
    from test_table_oracles import RUN_TIME_VALUE_CASES, RUN_TIME_VALUE_REQUEST, run_time_value_table, _cel_cases
    from cerbos_b200.table.bytecode import Unsupported
    now = parse_timestamp("2021-04-22T10:05:20.021-05:00")
    os.environ["CERBOS_B200_NO_JIT"] = "1"   # one table per expression: skip the background NVRTC compile (read at cgpu_init)
    from cerbos_b200 import capi
    ctx = capi.Context(0)
    try:
        cases = [(e, RUN_TIME_VALUE_REQUEST) for e in RUN_TIME_VALUE_CASES]
        for f, e, req in _cel_cases():
            if any(k in e for k in ("except", "intersect", "sort", "transform", ".map(", ".filter(", "split", "replace", "substring", "charAt", "indexOf",
                                    "Ascii", "trim", "reverse", "slice", "flatten", "lists.range", "hierarchy([", ")[", " + ", "spiffe")):
                inp = {"principal": dict(req.get("principal") or {}), "resource": dict(req.get("resource") or {}), "actions": ["a"]}
                inp["resource"]["kind"] = "leave_request"
                inp["principal"].setdefault("roles", ["r"])
                cases.append((e, inp))
        n = 0
        for e, inp in cases:
            try:
                rt, ft = run_time_value_table(e)
            except Unsupported:
                continue
            b = Encoder(ft.manifest).encode([inp])
            want = CheckOracle(rt).check(inp, now)["actions"]["a"]["effect"]
            t = ctx.load_table(ft.blob)
            got = t.check(b.columns, b.n, b.max_actions, now.ns)
            assert got[0, 0] == want, e
            t.release()
            n += 1
        assert n >= 98, n      # incl. the 18 SPIFFE leaves of the goldens
    finally:
        os.environ.pop("CERBOS_B200_NO_JIT", None)
        ctx.close()


def test_decision_metadata_on_gpu():
    """cgpu_check_meta through Engine.check(include_meta=True): effect, policy, scope of all 166 reference decisions and the
    effectiveDerivedRoles of every output, against the reference's own recorded answers (engine goldens)."""
    from cerbos_b200.engine import Engine
    from helpers import engine_decisions, load_golden
    docs = [e["policy"] for e in load_golden("store_policies.json")]
    engines = {False: Engine(docs, globals_={"environment": "test"}),
               True: Engine(docs, globals_={"environment": "test"}, lenient_scope_search=True)}
    n = n_edr = 0
    for cid, lenient, inp, want in engine_decisions():
        got = engines[lenient].check([inp], now_ns=NOW_NS, include_meta=True)[0]
        plain = engines[lenient].check([inp], now_ns=NOW_NS)[0]
        for a, wv in want["actions"].items():
            g = got["actions"][a]
            assert (g["effect"], g["policy"], g["scope"]) == (wv["effect"], wv.get("policy", ""), wv.get("scope", "")), (cid, a)
            assert plain["actions"][a]["effect"] == g["effect"], (cid, a)
            n += 1
        wedr = sorted(want.get("effectiveDerivedRoles", want.get("effective_derived_roles")) or [])
        assert got["effectiveDerivedRoles"] == wedr, cid
        n_edr += bool(wedr)
    assert n == 166 and n_edr >= 20
    for e in engines.values():
        e.close()


def test_multi_device_context_shards_a_batch():
    """cgpu_init with several devices in ONE process (SURVEY 8(b)): the table lives on every device, cgpu_check cuts the batch
    into one index range per device; results index-aligned and equal to the oracle.  Needs >= 2 GPUs."""
    import torch
    from cerbos_b200 import capi
    import workloads as W
    from oracle import cref
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs at least two GPUs")
    for name, n in (("C2", (1 << 18) + 999), ("C3", (1 << 17) + 3)):
        w = W.WORKLOADS[name]()
        _, ft, enc = W.build(w)
        b = w.columns(w.fields(n), enc)
        want = cref.check(ft.blob, b.columns, b.n, b.max_actions, n_threads=os.cpu_count() or 1)
        c = capi.Context(list(range(min(n_dev, 4))))
        t = c.load_table(ft.blob)
        t.wait_ready()
        for _ in range(2):
            assert (t.check(b.columns, b.n, b.max_actions) == want).all(), name
        t.release()
        c.close()


def test_fused_gather_against_nccl_under_torchrun():
    """tests/mgpu_gather_check.py (two ranks, one per GPU): the image gathered through cgpu_check_device_gather -- peer stores
    fused into the kernels -- must equal an NCCL all-gather of the plain path on every rank.  Needs two GPUs."""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29541", os.path.join(root, "tests", "mgpu_gather_check.py")], capture_output=True, text=True, timeout=900, cwd=root)
    assert r.returncode == 0 and "MGPU_GATHER_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
