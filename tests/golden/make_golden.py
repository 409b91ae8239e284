#!/usr/bin/env python3
"""Extracts the reference's golden TEST VECTORS for the CheckResources hot path
into compact JSON fixtures under tests/golden/.

Needs a cerbos/cerbos source tree (CERBOS_SRC, the directory holding internal/):
    python tests/golden/make_golden.py

Sources (all test data, no reference source code is copied):
  internal/test/testdata/cel_eval/*.yaml               -> cel_eval.json
      runner: internal/engine/evaluator_test.go:24-50 (now = 2021-04-22T10:05:20.021-05:00)
  internal/conditions/cerbos_lib_test.go:26-134 (expression table) -> cerbos_lib_test.json
  internal/test/testdata/engine/*.yaml,
  .../engine_strict_scope_search/*.yaml,
  .../engine_lenient_scope_search/*.yaml               -> engine_cases.json
      runner: internal/engine/engine_test.go:50-234 (globals {"environment":"test"},
      default version "default", default scope "")
  internal/test/testdata/store/**  (policies the engine goldens run against) -> store_policies.json
      loader skip rules: internal/util/filesystem.go:21-66,139-166,
      internal/storage/index/builder.go:105-144
  internal/test/testdata/server/checks/check_resources/*.yaml -> check_resources_cases.json
      (API-level goldens incl. JWT claims; JWTs are decoded here without verification)
"""
from __future__ import annotations

import base64
import json
import os
import re
import sys

import yaml

REF = os.path.join(os.environ.get("CERBOS_SRC", "."), "internal")
TD = f"{REF}/test/testdata"
OUT = os.path.dirname(os.path.abspath(__file__))


def load_yaml_docs(path):
    with open(path, encoding="utf-8") as f:
        text = f.read()
    docs = [d for d in yaml.safe_load_all(text) if d is not None]
    return docs


def dump(name, obj):
    p = os.path.join(OUT, name)
    with open(p, "w", encoding="utf-8") as f:
        json.dump(obj, f, indent=1, sort_keys=True, ensure_ascii=False)
        f.write("\n")
    print(f"wrote {p}: {len(obj) if hasattr(obj, '__len__') else ''}")


def cel_eval():
    out = []
    d = f"{TD}/cel_eval"
    for fn in sorted(os.listdir(d)):
        if not fn.endswith(".yaml"):
            continue
        doc = load_yaml_docs(f"{d}/{fn}")[0]
        out.append({"file": fn, "condition": doc["condition"], "request": doc["request"],
                    "want": bool(doc.get("want", False)), "wantError": bool(doc.get("wantError", False))})
    dump("cel_eval.json", out)


def cerbos_lib_table():
    src = open(f"{REF}/conditions/cerbos_lib_test.go", encoding="utf-8").read()
    start = src.index("func TestCerbosLib")
    end = src.index("env, err := cel.NewEnv", start)
    body = src[start:end]
    out = []
    for m in re.finditer(r"\{expr: `([^`]*)`(, wantErr: true)?\}", body):
        out.append({"expr": m.group(1), "wantErr": bool(m.group(2))})
    dump("cerbos_lib_test.json", out)


def engine_cases():
    out = []
    for sub, lenient in (("engine", False), ("engine_strict_scope_search", False),
                         ("engine_lenient_scope_search", True)):
        d = f"{TD}/{sub}"
        for fn in sorted(os.listdir(d)):
            if not fn.endswith((".yaml", ".yml", ".json")):
                continue
            doc = load_yaml_docs(f"{d}/{fn}")[0]
            out.append({"suite": sub, "file": fn, "lenient": lenient,
                        "description": doc.get("description", ""),
                        "inputs": doc.get("inputs", []), "wantOutputs": doc.get("wantOutputs", []),
                        "wantError": bool(doc.get("wantError", False))})
    dump("engine_cases.json", out)


_SUPPORTED_EXT = (".yaml", ".yml", ".json")


def store_policies():
    root = f"{TD}/store"
    out = []
    for dirpath, dirnames, filenames in os.walk(root):
        # skip rules: hidden dirs, _schemas, testdata
        dirnames[:] = sorted(x for x in dirnames if not x.startswith(".") and x not in ("_schemas", "testdata"))
        for fn in sorted(filenames):
            if fn.startswith(".") or not fn.endswith(_SUPPORTED_EXT):
                continue
            stem = fn.rsplit(".", 1)[0]
            if stem.endswith("_test"):
                continue
            rel = os.path.relpath(os.path.join(dirpath, fn), root)
            for doc in load_yaml_docs(os.path.join(dirpath, fn)):
                if not isinstance(doc, dict) or "apiVersion" not in doc:
                    continue
                out.append({"path": rel, "policy": doc})
    dump("store_policies.json", out)


def _jwt_claims(token: str):
    parts = token.split(".")
    if len(parts) != 3:
        return None
    pad = "=" * (-len(parts[1]) % 4)
    try:
        return json.loads(base64.urlsafe_b64decode(parts[1] + pad))
    except Exception:
        return None


def check_resources_cases():
    d = f"{TD}/server/checks/check_resources"
    out = []
    for fn in sorted(os.listdir(d)):
        if not fn.endswith(".yaml"):
            continue
        doc = load_yaml_docs(f"{d}/{fn}")[0]
        cr = doc.get("checkResources")
        if not cr:
            continue
        inp = cr.get("input", {})
        claims = None
        tok = ((inp.get("auxData") or {}).get("jwt") or {}).get("token")
        if tok:
            claims = _jwt_claims(tok)
        out.append({"file": fn, "description": doc.get("description", ""), "wantStatus": doc.get("wantStatus"),
                    "wantError": bool(doc.get("wantError", False)),
                    "input": inp, "jwtClaims": claims, "wantResponse": cr.get("wantResponse")})
    dump("check_resources_cases.json", out)



def verify_cases():
    """internal/test/testdata/verify/cases/case_*.yaml{.input,.golden}: policy test suites (txtar archives of fixtures +
    *_test.yaml files) run by the reference against the `store` policies; the .golden records, per test x principal x
    resource x action, what the ENGINE answered (success.effect, or failure.actual when the suite's expectation was
    wrong).  Those engine answers are emitted as (CheckInput, now, lenient, {action: effect}) vectors.
    Reference: internal/verify/verify_test.go:375-389 (store), internal/verify/test_fixture.go / test_suite_run.go."""
    import glob
    base = os.path.join(REF, "test/testdata/verify/cases")
    out = []
    for gpath in sorted(glob.glob(os.path.join(base, "*.golden"))):
        case = os.path.basename(gpath)[: -len(".golden")]
        try:
            golden = json.load(open(gpath))
        except ValueError:
            continue
        files, cur = {}, None
        for line in open(os.path.join(base, case + ".input")).read().split("\n"):
            if line.startswith("-- ") and line.endswith(" --"):
                cur = line[3:-3].strip()
                files[cur] = []
            elif cur is not None:
                files[cur].append(line)
        docs = {}
        for name, lines in files.items():
            try:
                docs[name] = yaml.safe_load("\n".join(lines)) if not name.endswith(".json") else json.loads("\n".join(lines))
            except Exception:
                docs[name] = None
        # fixtures: every testdata/* file may contribute principals / resources / auxData (+ groups)
        fx = {"principals": {}, "resources": {}, "auxData": {}, "principalGroups": {}, "resourceGroups": {}}
        for name, d in docs.items():
            if name.startswith("testdata/") and isinstance(d, dict):
                for k in fx:
                    if isinstance(d.get(k), dict):
                        fx[k].update(d[k])
        for s in golden.get("suites", []):
            suite = docs.get(s.get("file"))
            if not isinstance(suite, dict) or s.get("error"):
                continue
            loc = {k: dict(v) for k, v in fx.items()}
            for k in loc:
                if isinstance(suite.get(k), dict):
                    loc[k].update(suite[k])
            sopt = suite.get("options") or {}
            tests = {t.get("name"): t for t in (suite.get("tests") or []) if isinstance(t, dict)}
            for tc in s.get("testCases", []):
                t = tests.get(tc.get("name"))
                if t is None:
                    continue
                opt = {**sopt, **(t.get("options") or {})}
                inp = t.get("input") or {}
                aux = loc["auxData"].get(inp.get("auxData")) if inp.get("auxData") else None
                for pr in tc.get("principals", []):
                    principal = loc["principals"].get(pr["name"])
                    for rs in pr.get("resources", []):
                        resource = loc["resources"].get(rs["name"])
                        want = {}
                        for a in rs.get("actions", []):
                            det = a.get("details") or {}
                            eff = (det.get("success") or {}).get("effect") or (det.get("failure") or {}).get("actual")
                            if eff in ("EFFECT_ALLOW", "EFFECT_DENY"):
                                want[a["name"]] = eff
                        if not want or principal is None or resource is None:
                            continue
                        ci = {"requestId": f"{case}/{tc.get('name')}", "actions": list(want), "principal": principal, "resource": resource}
                        if aux:
                            ci["auxData"] = aux
                        out.append({"file": case, "suite": s.get("file"), "test": tc.get("name"), "now": opt.get("now"),
                                    "lenient": bool(opt.get("lenientScopeSearch")), "defaultPolicyVersion": opt.get("defaultPolicyVersion"),
                                    "defaultScope": opt.get("defaultScope"),
                                    "globals": opt.get("globals"), "input": ci, "want": want})
    dump("verify_cases.json", out)
    print("verify_cases:", len(out), "inputs,", sum(len(o["want"]) for o in out), "decisions")


def compile_cases():
    """internal/test/testdata/compile/*.yaml (+ .input): the compile front-end's own test cases -- a set of policy files
    and either the errors the reference's compiler reports for it or (no wantErrors) a successful compilation.  Kept: the
    files as parsed documents and the error kinds; the exact messages and source positions are presentation."""
    import re
    src = os.path.join(REF, "test/testdata/compile")
    out = []
    for name in sorted({f[:-5] for f in os.listdir(src) if f.endswith(".yaml")}):
        spec = [x for x in yaml.safe_load_all(open(os.path.join(src, name + ".yaml"))) if x][0]
        parts = re.split(r"^-- (.+?) --\s*$", open(os.path.join(src, name + ".yaml.input")).read(), flags=re.M)
        files = {parts[i]: [d for d in yaml.safe_load_all(parts[i + 1]) if d] for i in range(1, len(parts), 2)}
        out.append({"name": name, "mainDef": spec.get("mainDef"), "files": files,
                    "wantErrors": [{"file": e.get("file"), "error": e.get("error")} for e in (spec.get("wantErrors") or [])]})
    with open(os.path.join(OUT, "compile_cases.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True, default=str)
    print("compile cases:", len(out))


def ruletable_bundle():
    """internal/test/testdata/bundle/v2_ruletable/bundle_unencrypted.crrt: the reference compiler's own output for the
    `store` policies as a serialized runtimev1.RuleTable (what OpenRuleTableBundle unmarshals,
    internal/storage/hub/ruletable_bundle.go:36-87).  Kept verbatim: it pins cerbos_b200/table/ruletable_pb.py (bundle
    ingestion) and, row for row, cerbos_b200/policy/compile.py."""
    import shutil
    src = os.path.join(REF, "test/testdata/bundle/v2_ruletable/bundle_unencrypted.crrt")
    shutil.copyfile(src, os.path.join(OUT, "ruletable_bundle_unencrypted.crrt"))
    print("ruletable bundle:", os.path.getsize(src), "bytes")
    # the same rule table as the PDP receives it from Cerbos Hub: encrypted (bundle.crrts) + its key (encryption_key.txt);
    # pins cerbos_b200/table/bundle_crypto.py (crypto.DecryptChaCha20Poly1305Stream of github.com/cerbos/cloud-api)
    for name, out in (("bundle.crrts", "ruletable_bundle_encrypted.crrts"), ("encryption_key.txt", "ruletable_bundle_encryption_key.txt")):
        shutil.copyfile(os.path.join(REF, "test/testdata/bundle/v2_ruletable", name), os.path.join(OUT, out))


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("set CERBOS_SRC to a cerbos/cerbos source tree")
    cel_eval()
    cerbos_lib_table()
    engine_cases()
    store_policies()
    check_resources_cases()
    verify_cases()
    ruletable_bundle()
    compile_cases()
