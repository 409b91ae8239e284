"""The pipelined host-buffer check path (check_range): how it rejects a malformed narrow descriptor, and which kernels it
launches per chunk.

(a) Every defect of a narrow descriptor fails both narrow entry points with CGPU_ERR_INVALID before any device work,
    for an empty batch as well, and the context stays usable.
(b) Over a batch cut into chunks of 4096 requests, each of the five host-buffer entry points launches exactly the kernels
    its launch plan names, once per chunk, plus what the narrow form adds once per call."""
import ctypes

import numpy as np
import pytest

import workloads as W
from cerbos_b200 import meta as M
from cerbos_b200 import narrow as NW
from oracle.celeval import parse_timestamp

NOW_NS = parse_timestamp("2024-01-01T00:00:00Z").ns
CHUNK = 4096
N_CHUNKED = 3 * CHUNK + 77

_built = {}


def _workload(name):
    """-> (workload, rule table, FlatTable, Encoder), built once per module"""
    if name not in _built:
        w = W.WORKLOADS[name]()
        _built[name] = (w, *W.build(w))
    return _built[name]


def _batch(name, n):
    w, _, _, enc = _workload(name)
    return W.columns_parallel(w, n, 0, enc)


def _n_slots(name):
    return len(_workload(name)[3].slots)


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
            loaded[name].wait_ready()
        return loaded[name]
    yield get
    for t in loaded.values():
        t.release()


# ---- (a) invalid narrow descriptors --------------------------------------------------------------------------------------
def _classes(nr, cls, keep):
    arr = np.ascontiguousarray(cls, dtype=np.uint8)
    keep.append(arr)
    nr.slot_class = arr.ctypes.data


def _slot_class_above_u8_num(nr, classes, keep):
    c = classes.copy()
    c[0] = NW.SLOT_U8_NUM + 1
    _classes(nr, c, keep)


def _u16_id_without_slot_base(nr, classes, keep):
    c = classes.copy()
    c[0] = NW.SLOT_U16_ID
    _classes(nr, c, keep)
    nr.slot_base = None


def _hdr_const_mask_above_bit_3(nr, classes, keep):
    nr.hdr_const_mask |= 0x10


def _missing_hdr16(nr, classes, keep):
    nr.hdr_const_mask = 0
    nr.hdr16 = None


def _missing_versions(nr, classes, keep):
    nr.versions_const = 0
    nr.versions = None


def _missing_principal(nr, classes, keep):
    nr.principal_id = None
    nr.principal_id16 = None


def _heap_bits_8(nr, classes, keep):
    nr.heap_bits = 8


DEFECTS = {f.__name__.lstrip("_"): f for f in (_heap_bits_8, _slot_class_above_u8_num, _u16_id_without_slot_base, _hdr_const_mask_above_bit_3,
                                                 _missing_hdr16, _missing_versions, _missing_principal)}


def _wide_slots_table():
    """A table with 65 attribute slots: one more than the narrow wire carries."""
    from cerbos_b200.encode import Encoder
    from cerbos_b200.policy.compile import build_rule_table
    from cerbos_b200.table.flatten import flatten
    expr = " || ".join(f'R.attr.a{i} == "v{i}"' for i in range(65))
    pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "doc", "version": "default", "rules": [
        {"actions": ["a"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": expr}}}]}}
    ft = flatten(build_rule_table([pol]))
    enc = Encoder(ft.manifest)
    assert len(enc.slots) == 65
    b = enc.encode([{"actions": ["a"], "principal": {"id": "p", "roles": ["r"]},
                     "resource": {"kind": "doc", "id": str(i), "attr": {f"a{j}": f"v{j}" for j in range(i % 7, 65, 7)}}} for i in range(50)])
    nb = NW.narrow_batch(b, len(enc.slots))
    assert nb is not None
    return ft, nb


def _both_narrow_calls(ctx, t, bb, nr):
    """-> the return codes of cgpu_check_narrow and cgpu_check_narrow_meta on (bb, nr)"""
    from cerbos_b200 import capi
    L = capi.lib()
    n, km = bb.n_requests, max(bb.max_actions, 1)
    out = np.empty((max(n, 1), km), dtype=np.uint8)
    am = np.empty((max(n, 1), km), dtype=np.uint32)
    rm = np.empty(max(n, 1), dtype=M.REQUEST_META_DTYPE)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    return (L.cgpu_check_narrow(ctx._h, t._h, ctypes.byref(bb), ctypes.byref(nr), p(out)),
            L.cgpu_check_narrow_meta(ctx._h, t._h, ctypes.byref(bb), ctypes.byref(nr), p(out), p(am), p(rm)))


def _empty(bb):
    from cerbos_b200 import capi
    return capi._Batch(0, bb.max_actions, bb.now_unix_nanos, bb.flags, bb.columns, bb.column_bytes, bb.n_columns)


def _assert_rejected_then_usable(ctx, tables, t, bb, nr, what):
    from cerbos_b200 import capi
    assert _both_narrow_calls(ctx, t, bb, nr) == (capi.ERR_INVALID, capi.ERR_INVALID), what
    # the context is still usable: a valid call right behind the rejected ones
    good = _batch("C3", 1000)
    nb = NW.narrow_batch(good, _n_slots("C3"))
    c3 = tables("C3")
    assert (c3.check_narrow(nb, NOW_NS) == c3.check(good.columns, good.n, good.max_actions, NOW_NS)).all(), what


@pytest.mark.gpu
@pytest.mark.parametrize("empty", [False, True])
@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_invalid_narrow_descriptor(ctx, tables, defect, empty):
    """Each defect of the descriptor fails cgpu_check_narrow and cgpu_check_narrow_meta with CGPU_ERR_INVALID, also on an
    empty batch; the next valid call on the context succeeds."""
    from cerbos_b200 import capi
    t = tables("C3")
    nb = NW.narrow_batch(_batch("C3", 1000), _n_slots("C3"))
    bb, nr, keep = t.prepare_narrow(nb, NOW_NS)
    bad = capi._Narrow.from_buffer_copy(nr)
    DEFECTS[defect](bad, np.asarray(nb.slot_class, dtype=np.uint8), keep)
    _assert_rejected_then_usable(ctx, tables, t, _empty(bb) if empty else bb, bad, (defect, empty))
    del keep


@pytest.mark.gpu
@pytest.mark.parametrize("empty", [False, True])
def test_too_many_slots_for_the_narrow_wire(ctx, tables, empty):
    """A table with more than 64 attribute slots cannot take a narrow batch: CGPU_ERR_INVALID from both entry points."""
    ft, nb = _wide_slots_table()
    t = ctx.load_table(ft.blob)
    try:
        bb, nr, keep = t.prepare_narrow(nb, NOW_NS)
        _assert_rejected_then_usable(ctx, tables, t, _empty(bb) if empty else bb, nr, ("65 slots", empty))
        del keep
    finally:
        t.release()


# ---- (b) launch counts ---------------------------------------------------------------------------------------------------
def _launches(ctx, call):
    before = ctx.launch_count()
    call()
    return ctx.launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C3", "C5"])
def test_launches_per_chunk(ctx, tables, name, monkeypatch):
    """One call of each host-buffer entry point over 4 chunks launches, per chunk, the kernels of its plan:
    - effects: the check kernel, the lean body's drain, and the plan's pre-passes (merged rows, string predicates);
    - metadata: the same pre-passes, the metadata form of the unique-condition kernel and its reference-order drain, or
      the reference-order body alone on a table without the unique-condition path;
    - rule outputs: the reference-order output body;
    and the narrow form adds one widening launch per chunk and one for a narrowed heap per call."""
    t = tables(name)
    b = _batch(name, N_CHUNKED)
    nb = NW.narrow_batch(b, _n_slots(name))
    assert nb is not None
    n_chunks = -(-N_CHUNKED // CHUNK)
    widen = n_chunks + (1 if (nb.heap_u32 or nb.heap_bits == 16) and np.asarray(nb.tables[0]).nbytes else 0)

    def wide():
        return t.check(b.columns, b.n, b.max_actions, NOW_NS)

    # the effect plan (the same for every chunk: index order, no clustering below 32768 requests), and its pre-passes,
    # the launches of one single-chunk call beyond the check kernel and the drain
    one = _launches(ctx, wide)
    cfg = ctx.last_kernel_config()
    assert not cfg["clustered"], cfg
    lean, uc = int(cfg["lean_body"]), int(cfg["unique_conditions"])
    pre = one - 1 - lean
    assert 0 <= pre <= 2 * uc, (one, cfg)

    monkeypatch.setenv("CERBOS_B200_CHECK_CHUNK", str(CHUNK))
    effects = 1 + lean + pre
    assert _launches(ctx, wide) == n_chunks * effects, cfg
    assert _launches(ctx, lambda: t.check_narrow(nb, NOW_NS)) == n_chunks * effects + widen, cfg

    got = _launches(ctx, lambda: t.check_meta(b.columns, b.n, b.max_actions, NOW_NS))
    meta_uc = ctx.last_kernel_config()["unique_conditions"]   # the effect plan's kernel in metadata form, where the table has its side table
    assert uc or not meta_uc, cfg
    meta = pre + 2 if meta_uc else 1
    assert got == n_chunks * meta, (got, cfg)
    assert _launches(ctx, lambda: t.check_narrow_meta(nb, NOW_NS)) == n_chunks * meta + widen, cfg

    assert _launches(ctx, lambda: t.check_outputs(b.columns, b.n, b.max_actions, 64, NOW_NS)) == n_chunks, cfg
    assert ctx.last_kernel_config()["grid"] >= 1
