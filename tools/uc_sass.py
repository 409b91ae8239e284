#!/usr/bin/env python3
"""What the unique-condition kernels of one workload compile to, without a device.

Generates the workload table's run-time specialised translation unit and compiles it with NVRTC exactly as a table
load does (capi.compile_check), then prints for cb_spec_uc / cb_spec_uc_global and their metadata forms: registers and stack, the SASS
instruction count, the part of it inlined from cb::eval_request_uc (the per-request path), the generic byte loads
(LD.E.U8), the local-memory loads and stores (LDL / STL) and the instruction count per source function (the innermost function of each instruction's line info,
nvdisasm -gi).  Needs the built library and the CUDA toolkit's cuobjdump / nvdisasm.

    python tools/uc_sass.py C3                    # the build as it is
    python tools/uc_sass.py C3 --defs -DCB_UC_STUB_TERMS
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("cb_spec_uc", "cb_spec_uc_global", "cb_spec_uc_meta", "cb_spec_uc_meta_global")
_DEF = re.compile(r"^\s*(?:template\s*<[^>]*>\s*)?(?:static\s+)?(?:CB_HD_NOINLINE|CB_HD|__device__[\w\s]*|inline)\b[^;=]*?(\boperator\(\)|\b\w+)\s*\(")
_LINE = re.compile(r'//## File "[^"]*", line (\d+)')
_INSN = re.compile(r"^\s+/\*[0-9a-f]+\*/\s+(.*?)\s*;")


def tool(name):
    for d in (os.environ.get("CUDA_HOME", ""), "/usr/local/cuda"):
        p = os.path.join(d, "bin", name)
        if d and os.path.exists(p):
            return p
    return name


def function_of_line(tu_lines):
    """line number (1-based) -> name of the function whose body holds it (nearest definition above)."""
    names, cur = [None], None
    for text in tu_lines:
        m = _DEF.match(text)
        if m and not text.rstrip().endswith(";"):
            cur = m.group(1)
        names.append(cur)
    return names


def analyse(sass, fname, kernel):
    """-> dict for one kernel of the nvdisasm -gi listing."""
    start = sass.find(f"\n.text.{kernel}:")
    if start < 0:
        return None
    end = sass.find("\n.text.", start + 1)
    body = sass[start:end if end > 0 else len(sass)].splitlines()
    per_fn = collections.Counter()
    total = req = u8 = ldl = stl = 0
    chain, fresh = [], False
    for text in body:
        m = _LINE.search(text)
        if m:
            if not fresh:
                chain = []
                fresh = True
            chain.append(int(m.group(1)))
            continue
        ins = _INSN.match(text)
        if not ins:
            continue
        fresh = False
        op = ins.group(1).split()
        op = op[1] if op and op[0].startswith("@") and len(op) > 1 else (op[0] if op else "")
        if op == "NOP":
            continue
        total += 1
        u8 += op.startswith("LD.E.U8")
        ldl += op.startswith("LDL")
        stl += op.startswith("STL")
        fns = [fname[n] if n < len(fname) else None for n in chain]
        if "eval_request_uc" in fns:
            req += 1
        per_fn[fns[0] if fns else None] += 1
    return {"total": total, "request_path": req, "ld_e_u8": u8, "ldl": ldl, "stl": stl, "per_fn": per_fn}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("workload", nargs="?", default="C3")
    ap.add_argument("--defs", default="", help="extra -D options for the generated unit (CERBOS_B200_SPEC_DEFS)")
    ap.add_argument("--top", type=int, default=25, help="source functions listed per kernel")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["CERBOS_B200_CACHE_DIR"] = tmp          # the compiled cubin lands here, not in the user's cache
        os.environ["CERBOS_B200_SPEC_DUMP"] = os.path.join(tmp, "tu.cu")
        os.environ["CERBOS_B200_SPEC_DEFS"] = a.defs
        import workloads as W
        from cerbos_b200 import capi
        w = W.WORKLOADS[a.workload]()
        _, ft, _ = W.build(w)
        n, note = capi.compile_check(ft.blob)
        cubins = [f for f in os.listdir(tmp) if f.endswith(".cubin")]
        if not n or not cubins:
            sys.exit(f"{a.workload}: no specialised unit ({note})")
        cubin = os.path.join(tmp, cubins[0])
        with open(os.path.join(tmp, "tu.cu")) as f:
            fname = function_of_line(f.read().splitlines())
        res = subprocess.run([tool("cuobjdump"), "-res-usage", cubin], capture_output=True, text=True, check=True).stdout
        sass = subprocess.run([tool("nvdisasm"), "-gi", "-c", cubin], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\w+):\s*\n\s*(REG:\d+ STACK:\d+)", res))
    print(f"{a.workload} {a.defs or '(no extra defines)'}")
    for k in KERNELS:
        r = analyse(sass, fname, k)
        if r is None:
            print(f"{k}: not in this unit")
            continue
        print(f"{k}: {usage.get(k, '?')}  instructions {r['total']}  per-request path (eval_request_uc) {r['request_path']}  LD.E.U8 {r['ld_e_u8']}  LDL {r['ldl']}  STL {r['stl']}")
        for fn, c in r["per_fn"].most_common(a.top):
            print(f"    {c:6d}  {fn}")


if __name__ == "__main__":
    main()
