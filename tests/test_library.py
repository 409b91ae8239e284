"""The C-ABI library loads and exports every symbol include/cerbos_b200.h declares (no compute without a GPU)."""
import os
import re

import pytest

from cerbos_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_match_header():
    hdr = open(os.path.join(ROOT, "include", "cerbos_b200.h")).read()
    declared = set(re.findall(r"\b(cgpu_[a-z_]+)\s*\(", hdr))
    assert declared == set(capi.EXPORTS), declared ^ set(capi.EXPORTS)
    lib = capi.lib()
    for name in declared:
        assert hasattr(lib, name), name


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(capi.CgpuError) as e:
        capi.Context(0)
    assert e.value.code == capi.ERR_NO_DEVICE


def test_product_does_not_import_oracle():
    """Nothing under cerbos_b200/ may import or reference the oracle (test infrastructure)."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "cerbos_b200")):
        for fn in files:
            if fn.endswith((".py", ".cu", ".h", ".cpp")):
                src = open(os.path.join(dirpath, fn), encoding="utf-8").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), os.path.join(dirpath, fn)
                assert "check_ref" not in src, os.path.join(dirpath, fn)


def test_runtime_specialisation_compiles_without_a_device():
    """The table-specialised translation unit the library hands to NVRTC at table load (embedded cb_core.h / cb_kernels.h +
    generated block evaluators, or -- tables with many block shapes -- the unique-condition evaluator) compiles for sm_90a
    here, without a GPU -- C5 too (73 distinct conditions, 50 of them leaf programs translated from their bytecode); tables
    that do not qualify say why (a condition building a list in the arena: no translation)."""
    from cerbos_b200 import capi
    from cerbos_b200.policy.compile import build_rule_table
    from cerbos_b200.table.flatten import flatten
    import workloads as W
    for name in ("C1", "C2", "C3", "C5"):
        _, ft, _ = W.build(W.WORKLOADS[name]())
        n, note = capi.compile_check(ft.blob)
        assert n > 10000 and note == "ok", (name, n, note)
    rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}}
             for i, e in enumerate(['P.attr.teams.map(t, t + "!") == ["x!"]'] + [f'R.attr.v{i} == {i}' for i in range(12)])]
    docs = [{"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": f"k{j}", "version": "default", "rules": rules[j:] + rules[:j]}} for j in range(12)]
    n, note = capi.compile_check(flatten(build_rule_table(docs)).blob)
    assert n == 0 and "does not qualify" in note, (n, note)
