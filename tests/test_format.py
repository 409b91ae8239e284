"""ext.Strings `format` and `strings.quote` on the device (table/bytecode.py FORMAT / FN QUOTE, cb_core.h op_format / str_quote).

Oracle #1 (oracle/celeval.py: _str_format, _fmt_verb, _fmt_s, format_double, _f_quote) is the specification.  Checked here:
  * the number printers of cb_core.h, compiled for the host: shortest round-trip digits (Schubfach) against oracle #1's
    format_double, %.{p}f / %.{p}e for p = 0..20 against the C library's and Python's exactly rounded formatting;
  * the power table of the shortest-digit printer, recomputed with exact integer arithmetic;
  * a documentation row and the reference's golden rule outputs that call format, as conditions;
  * written-out cases on every verb and argument type (and their negations), through oracle #1, the interpreter and the
    generated leaf programs;
  * a seeded differential run of random format / quote expressions over requests whose attributes change type;
  * the build-time side (constant format strings only, leaf-program translation, the NVRTC unit);
  * on the GPU: the NVRTC kernel, the general kernel and the narrow wire path against oracle #1."""
import json
import os
import random
import struct
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table import layout as L
from cerbos_b200.table.bytecode import Unsupported
from cerbos_b200.table.flatten import flatten
from helpers import load_golden
from hostsim import driver as hostsim
from oracle import cref
from oracle.celeval import format_double, parse_timestamp
from oracle.check import CheckOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOW = parse_timestamp("2021-04-22T10:05:20.021-05:00")

PRINTERS = r"""
#include <cstdint>
#include <cstdio>
#include <cstring>
#include "cb_core.h"
using namespace cb;
// stdin: doubles, 8 bytes each.  g: the %s text of each (shortest digits), one per line.  fe: %.pf and %.pe for p = 0..20
// against the C library's (exactly rounded, ties to even), then "<doubles> <mismatches>".  dump: those 42 texts per double.
static Ctx ctx;
int main(int argc, char **argv) {
    const char *mode = argv[1];
    uint64_t bits, n = 0, bad = 0;
    static char ref[4096];
    while (fread(&bits, 8, 1, stdin) == 1) {
        n++;
        double d;
        memcpy(&d, &bits, 8);
        if (!strcmp(mode, "g")) {
            ctx.scr_used = 0;
            StrB s = strb_begin(ctx);
            put_double_g(s, bits);
            fwrite(reinterpret_cast<const char *>(ctx.scratch) + s.b0, 1, s.len, stdout);
            fputc('\n', stdout);
            continue;
        }
        for (int p = 0; p <= 20; p++)
            for (int e = 0; e < 2; e++) {
                ctx.scr_used = 0;
                StrB s = strb_begin(ctx);
                if (e) put_sci(s, bits, p); else put_fixed(s, bits, p);
                const char *t = reinterpret_cast<const char *>(ctx.scratch) + s.b0;
                if (!strcmp(mode, "dump")) { fwrite(t, 1, s.len, stdout); fputc('\n', stdout); continue; }
                const int rl = snprintf(ref, sizeof ref, e ? "%.*e" : "%.*f", p, d);
                if (!s.ok || (uint32_t)rl != s.len || memcmp(ref, t, s.len)) {
                    if (bad++ < 10) printf("mismatch %016llx %%.%d%c: %.*s / %s\n", (unsigned long long)bits, p, e ? 'e' : 'f', (int)s.len, t, ref);
                }
            }
    }
    if (!strcmp(mode, "fe")) printf("%llu %llu\n", (unsigned long long)n, (unsigned long long)bad);
    return 0;
}
"""


@pytest.fixture(scope="module")
def printers(tmp_path_factory):
    d = tmp_path_factory.mktemp("printers")
    src = d / "printers.cpp"
    src.write_text(PRINTERS)
    exe = str(d / "printers")
    subprocess.run(["g++", "-O2", "-std=c++17", f"-I{ROOT}/include", f"-I{ROOT}/cerbos_b200/csrc", "-o", exe, str(src)], check=True)
    return exe


def _bits(xs):
    return np.array([struct.unpack("<Q", struct.pack("<d", x))[0] for x in xs], dtype=np.uint64)


SPECIAL = [5e-324, 1e-323, 1.5e-323, 2.2250738585072014e-308, 2.225073858507201e-308, 1.7976931348623157e308, 1e23, 0.0, -0.0,
           9007199254740991.0, 9007199254740992.0, 9007199254740993.0, 9007199254740994.0, 9007199254740996.0,
           0.1, 0.3, 2.5, 123456.0, 1234567.0, 1e-5, 1e-4, 0.125, 0.375, 3.5, -2.5] + \
          [10.0 ** k for k in range(-30, 31)] + [float(f"1e{k}") for k in range(-30, 31)]


def _double_set(n, seed):
    """random bit patterns, random subnormals, every power of two and the special values; finite ones only"""
    rng = np.random.default_rng(seed)
    b = np.concatenate([_bits(SPECIAL), rng.integers(0, 2 ** 64, size=n, dtype=np.uint64),
                        rng.integers(1, 2 ** 52, size=n // 100, dtype=np.uint64) | (rng.integers(0, 2, size=n // 100, dtype=np.uint64) << 63),
                        np.arange(1, 2047, dtype=np.uint64) << 52])
    return b[np.isfinite(b.view(np.float64))]


def test_shortest_digits_match_oracle_format_double(printers):
    b = _double_set(1_000_000, 1)
    assert len(b) >= 1_000_000
    out = subprocess.run([printers, "g"], input=b.tobytes(), capture_output=True, check=True).stdout.decode().split("\n")[:-1]
    assert len(out) == len(b)
    bad = [(x, o) for x, o in zip(b.view(np.float64).tolist(), out) if format_double(x) != o]
    assert not bad, bad[:10]
    assert out[:3] == ["5e-324", "1e-323", "1.5e-323"] and out[SPECIAL.index(1e23)] == "1e+23"


def test_fixed_and_exponent_forms_are_exactly_rounded(printers):
    """%.{p}f / %.{p}e, p = 0..20, on 10^6 doubles against the C library (exact, ties to even on the binary value)"""
    b = _double_set(1_000_000, 2)
    chunks = np.array_split(b, os.cpu_count() or 1)

    def run(c):
        return subprocess.run([printers, "fe"], input=c.tobytes(), capture_output=True, check=True).stdout.decode()
    with ThreadPoolExecutor(len(chunks)) as ex:
        outs = list(ex.map(run, chunks))
    total = 0
    for o in outs:
        n, bad = map(int, o.strip().split("\n")[-1].split())
        assert bad == 0, o
        total += n
    assert total == len(b) >= 1_000_000


def test_fixed_and_exponent_forms_match_python(printers):
    """the same printers against Python's formatting on a sample, and on exact halfway cases"""
    b = np.concatenate([_double_set(20_000, 3), _bits([0.125, 0.375, 2.5, 3.5, -0.5, 1.5, 0.5])])
    out = subprocess.run([printers, "dump"], input=b.tobytes(), capture_output=True, check=True).stdout.decode().split("\n")[:-1]
    it = iter(out)
    for x in b.view(np.float64).tolist():
        for p in range(21):
            assert next(it) == f"{x:.{p}f}", (x, p)
            assert next(it) == f"{x:.{p}e}", (x, p)
    halves = dict(zip([0.125, 0.375, 2.5, 3.5], out[-7 * 42: -3 * 42: 42]))
    assert halves == {0.125: "0", 0.375: "0", 2.5: "2", 3.5: "4"}
    assert out[-7 * 42 + 4] == "0.12" and out[-6 * 42 + 4] == "0.38"    # %.2f: ties to even


def test_schubfach_power_table():
    """every entry of cb_core.h's CB_SCHUBFACH_G: g(k) = floor(10^-k / 2^r) + 1, 2^125 < g <= 2^126, split at bit 63"""
    text = open(os.path.join(ROOT, "cerbos_b200", "csrc", "cb_core.h")).read()
    body = text[text.index("#define CB_SCHUBFACH_G"):]
    body = body[:body.index("\n#if")]
    words = [int(w, 16) for w in body.replace("ull", "").replace("\\", "").split("CB_SCHUBFACH_G")[1].replace(",", " ").split()]
    assert len(words) == 2 * 617
    for i, e in enumerate(range(-292, 325)):     # e = -k
        fl = (10 ** e).bit_length() - 1 if e >= 0 else -(10 ** -e).bit_length()     # floor(log2 10^e)
        assert (e * 913124641741) >> 38 == fl
        r = fl - 125
        g = (10 ** e >> r if r >= 0 else 10 ** e << -r) + 1 if e >= 0 else (1 << (-r)) // 10 ** -e + 1
        assert 2 ** 125 < g <= 2 ** 126
        assert words[2 * i] == g >> 63 and words[2 * i + 1] == g & (2 ** 63 - 1), e


# ---- the kernel core -----------------------------------------------------------------------------------------------------
def _table(exprs):
    """one rule per expression, action a<i>"""
    rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}} for i, e in enumerate(exprs)]
    pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "leave_request", "version": "default", "rules": rules}}
    rt = build_rule_table([pol])
    return rt, flatten(rt)


def _kernel_core(rt, ft, reqs, tmp_path, programs=True):
    """decisions of oracle #1, the interpreter (general body) and -- programs: the generated leaf programs must exist --
    the host build of the unique-condition body with the generated code; all three must agree"""
    b = Encoder(ft.manifest).encode(reqs)
    n, k = b.n, b.max_actions
    o = CheckOracle(rt)
    want = np.array([[{"EFFECT_ALLOW": 1, "EFFECT_DENY": 2, 1: 1, 2: 2}[o.check(r, NOW)["actions"][a]["effect"]] for a in r["actions"]] for r in reqs], dtype=np.uint8)
    got = hostsim.check(ft.blob, b.columns, n, k, NOW.ns, mode=1)
    assert (got == want).all(), np.argwhere(got != want)[:8].tolist()
    src, _ = hostsim.generate_uc(ft.blob)
    if programs:
        assert "CB_HD bool uc_atom_" in src
        lib = hostsim.build_spec(ft.blob, str(tmp_path), uc=True)
        spec = hostsim.check_spec(lib, ft.blob, b.columns, n, k, NOW.ns, mode=4)
        assert (spec == want).all(), np.argwhere(spec != want)[:8].tolist()
    return want


REQUEST = {"principal": {"id": "john", "roles": ["employee"],
                         "attr": {"n": 12, "x": 2.5, "tiny": 1e-7, "big": 1.5e300, "neg": -0.0, "dept": "marketing", "esc": "a\"b\\c\n\té世\U0001F600",
                                  "ctl": "\u0007\u0008\u000c\r\u000b", "teams": ["design", "product"], "nested": [[1, "a"], {"k": [True, None]}],
                                  "m": {"b": 2, "a": 1.5, "c": "x"}, "ts": "2021-04-20T10:00:20.021-05:00", "ts0": "2021-04-20T10:00:20Z",
                                  "d": "-1h30m0.5s", "big_list": list(range(40)), "wide": {f"k{i}": i for i in range(17)}}},
           "resource": {"kind": "leave_request", "id": "r1", "attr": {"args": ["x", 3.25], "s": "héllo"}}}

# (expression, holds): None = the evaluation fails, so the expression and its negation are both denied
FORMAT_CASES = [
    # %s of every argument type
    ('"%s|%s|%s|%s|%s".format([null, true, false, 12, -7]) == "null|true|false|12|-7"', True),
    ('"%s %s %s".format([P.attr.n, P.attr.x, P.attr.tiny]) == "12 2.5 1e-07"', True),
    ('"%s %s".format([P.attr.big, 123456789.0]) == "1.5e+300 1.23456789e+08"', True),
    ('"%s %s %s".format([0.0 / 0.0, 1.0 / 0.0, -1.0 / 0.0]) == "NaN Infinity -Infinity"', True),
    ('"%s".format([P.attr.neg]) == "-0" && "%s".format([100000.0]) == "100000" && "%s".format([1000000.0]) == "1e+06"', True),
    ('"%s %s".format([3u, b"bytes"]) == "3 bytes"', True), ('"%s".format([base64.decode("/w==")]) == "x"', None),
    ('"%s".format([timestamp(P.attr.ts)]) == "2021-04-20T15:00:20.021Z" && "%s".format([timestamp(P.attr.ts0)]) == "2021-04-20T10:00:20Z"', True),
    ('"%s".format([duration(P.attr.d)]) == "-5400.5s" && "%s".format([duration("0s")]) == "0s" && "%s".format([duration("1.5ms")]) == "0.0015s"', True),
    ('"%s %s %s".format([type(1), type(P.attr.x), type(duration("1s"))]) == "int double google.protobuf.Duration"', True),
    ('"%s".format([P.attr.teams]) == "[design, product]" && "%s".format([[]]) == "[]"', True),
    ('"%s".format([P.attr.nested]) == "[[1, a], {k: [true, null]}]"', True),
    ('"%s".format([P.attr.m]) == "{a: 1.5, b: 2, c: x}" && "%s".format([{}]) == "{}"', True),
    ('"%s".format([{2: "x", 10: "y", "1": true}]) == "{1: true, 10: y, 2: x}"', True),
    ('"%s".format([P.attr.nope]) == "x"', None), ('"%s %s".format(["only one"]) == "x"', None),
    ('"%s".format(R.attr.args) == "x" && "%s-%s".format(R.attr.args) == "x-3.25"', True), ('"%s".format(P.attr.dept) == "x"', None),
    ('"no clauses %%".format([]) == "no clauses %" && "x".format([1, 2]) == "x"', True),
    # %d
    ('"%d %d %d".format([12, -9223372036854775807 - 1, 18446744073709551615u]) == "12 -9223372036854775808 18446744073709551615"', True),
    ('"%d %d".format([0.0 / 0.0, -1.0 / 0.0]) == "NaN -Infinity"', True), ('"%d".format([P.attr.n]) == "12"', None), ('"%d".format([true]) == "1"', None),
    ('"%d".format(["1"]) == "1"', None),
    # %f / %e with and without precision
    ('"%f %.2f %.0f %.0f".format([P.attr.x, 0.125, 2.5, 3.5]) == "2.500000 0.12 2 4"', True),
    ('"%.3f|%.1f|%f".format([-0.0005, P.attr.neg, 7]) == "-0.001|-0.0|7.000000"', True),
    ('"%e|%.2e|%.0e".format([P.attr.x, 123456.0, 9.5]) == "2.500000e+00|1.23e+05|1e+01"', True),
    ('"%.3e %e".format([P.attr.tiny, 5e-324]) == "1.000e-07 4.940656e-324"', True),
    ('"%f %e".format([0.0 / 0.0, 1.0 / 0.0]) == "NaN Infinity" && "%.2f".format([3u]) == "3.00"', True),
    ('"%.10f".format([0.1]) == "0.1000000000" && "%.20f".format([0.1]) == "0.10000000000000000555"', True),
    ('"%f".format(["1.0"]) == "x"', None), ('"%e".format([true]) == "x"', None), ('"%f".format([null]) == "x"', None),
    ('size("%f".format([P.attr.big])) == 308', True),
    # %b %o %x %X
    ('"%b %b %b %b".format([5, -5, true, 6u]) == "101 -101 1 110"', True), ('"%b".format([1.0]) == "1"', None),
    ('"%o %o %o".format([8, -8, 8u]) == "10 -10 10"', True), ('"%o".format(["8"]) == "x"', None),
    ('"%x %X %x %X".format([255, 255, -255, 3000000000u]) == "ff FF -ff B2D05E00"', True),
    ('"%x|%X|%x".format(["héllo", b"\\x01\\x7f", ""]) == "68c3a96c6c6f|017F|"', True), ('"%x".format([1.5]) == "x"', None), ('"%x".format([true]) == "x"', None),
    ('"%.3s %.9d".format(["abc", 5]) == "abc 5"', True),
    # malformed clauses: an error whatever the arguments are
    ('"%".format([1]) == "x"', None), ('"%z".format([1]) == "x"', None), ('"a%".format([]) == "a"', None),
    # strings.quote
    ('strings.quote(P.attr.esc) == "\\"a\\\\\\"b\\\\\\\\c\\\\n\\\\té世\U0001F600\\""', True),
    ('strings.quote(P.attr.ctl) == "\\"\\\\a\\\\b\\\\f\\\\r\\\\v\\""', True),
    ('strings.quote("") == "\\"\\"" && strings.quote(R.attr.s) == "\\"héllo\\""', True), ('strings.quote(P.attr.n) == "x"', None),
    # values flowing on
    ('"id:%s".format([P.id]) + "/" + "%d".format([size(P.attr.teams)]) == "id:john/2"', True),
    ('"%s-%s".format([P.attr.dept, R.id]).startsWith("marketing-r") && "%s".format([P.attr.dept]) == P.attr.dept', True),
    ('"%s".format(["%d"]) == "%d"', True),
]


def _pairs(cases):
    exprs, holds = [], []
    for e, h in cases:
        for neg in (False, True):
            exprs.append(f"!({e})" if neg else e)
            holds.append(h is not None and h != neg)
    return exprs, holds


def test_written_out_cases(tmp_path):
    """each case and its negation, 16 rules per table: oracle #1 gives the written answer, the interpreter and the generated
    leaf programs give oracle #1's"""
    exprs, holds = _pairs(FORMAT_CASES)
    for lo in range(0, len(exprs), 32):
        part = exprs[lo:lo + 32]
        rt, ft = _table(part)
        req = dict(REQUEST, actions=[f"a{i}" for i in range(len(part))])
        sub = tmp_path / str(lo)
        sub.mkdir()
        want = _kernel_core(rt, ft, [req], sub)
        for i, e in enumerate(part):
            assert want[0, i] == (1 if holds[lo + i] else 2), e
    # oracle #2 does not port value-building functions: it flags the new ops instead of misreading them
    rt, ft = _table(['"%s".format([P.id]) == "john"'])
    with pytest.raises(RuntimeError, match="-2"):
        cref.check(ft.blob, Encoder(ft.manifest).encode([dict(REQUEST, actions=["a0"])]).columns, 1, 1, NOW.ns)
    rt, ft = _table(['strings.quote(P.id) == "x"'])
    with pytest.raises(RuntimeError, match="-2"):
        cref.check(ft.blob, Encoder(ft.manifest).encode([dict(REQUEST, actions=["a0"])]).columns, 1, 1, NOW.ns)


@pytest.mark.parametrize("expr", [
    '"%s".format([P.attr.big_list.map(x, P.attr.big_list)]) == "x"',       # text larger than the scratch arena
    '"%.2000f".format([1.5]) == "x"',
    '"%s".format([P.attr.wide]) == "x"',                                  # a map of more than 16 entries
    '"%s".format([[[[[[1]]]]]]) == "x"',                                  # nested deeper than four containers
])
def test_what_the_device_cannot_print_is_flagged(expr):
    rt, ft = _table([expr])
    req = dict(REQUEST, actions=["a0"])
    b = Encoder(ft.manifest).encode([req])
    assert CheckOracle(rt).check(req, NOW)["actions"]["a0"]["effect"] in (1, 2, "EFFECT_ALLOW", "EFFECT_DENY")
    with pytest.raises(RuntimeError, match="-2"):
        hostsim.check(ft.blob, b.columns, 1, 1, NOW.ns, mode=1)


def test_documentation_row(tmp_path):
    rt, ft = _table(['"department_%s_%d".format(["marketing", 1]) == "department_marketing_1"'])
    assert (_kernel_core(rt, ft, [dict(REQUEST, actions=["a0"])], tmp_path) == 1).all()


def _golden_output_conditions():
    """(condition, request): `(<expr>) == <golden value>` for every rule output of the reference's golden store that calls
    format, over each golden request whose response carries that value"""
    from cerbos_b200.cel.parser import parse
    from oracle.activation import build_activation, build_request
    from oracle.celeval import eval_expr
    exprs = set()

    def walk(x):
        if isinstance(x, dict):
            for k, v in x.items():
                if k in ("expr", "ruleActivated", "conditionNotMet") and isinstance(v, str) and ".format(" in v:
                    exprs.add(v)
                walk(v)
        elif isinstance(x, list):
            for v in x:
                walk(v)
    walk([p for p in load_golden("store_policies.json")])
    pairs = []     # (request, response entry carrying `outputs`)
    for c in load_golden("check_resources_cases.json"):
        inp = c["input"]
        for res, r in zip((c.get("wantResponse") or {}).get("results") or [], inp.get("resources") or []):
            pairs.append(({"principal": inp["principal"], "resource": r["resource"]}, res))
    for c in load_golden("engine_cases.json"):
        for inp, res in zip(c.get("inputs") or [], c.get("wantOutputs") or []):
            pairs.append(({"principal": inp["principal"], "resource": inp["resource"]}, res))
    out = []
    for req, res in pairs:
        for o in res.get("outputs") or []:
            lit = json.dumps(o["val"])
            for e in sorted(exprs):
                cond = f"({e}) == {lit}"
                try:
                    ok = eval_expr(parse(cond), build_activation(build_request(req)), NOW) is True
                except Exception:  # noqa: BLE001 -- an expression over another request's attributes
                    ok = False
                if ok:
                    out.append((e, cond, req))
    return exprs, out


def test_golden_outputs_that_call_format(tmp_path):
    exprs, conds = _golden_output_conditions()
    # three output expressions call format; two of them have golden values (the approval_status output never fires there)
    assert len(exprs) == 3 and len({e for e, _, _ in conds}) == 2, (exprs, [e for e, _, _ in conds])
    assert not any("approval_status" in e for e, _, _ in conds)
    for i, (e, cond, req) in enumerate(conds):
        if e.lstrip().startswith("{"):
            # the map-valued output: its literal needs a deeper evaluation stack than the device has, so its format calls are
            # checked where they stand in the golden map
            lit = cond[len(f"({e}) == "):]
            cond = (f'{lit}["formatted_%s".format(["string"])] == "id:%s".format([P.id]) && '
                    f'{lit}["something_nested"]["nested_formatted_%s".format(["string"])] == "id:%s".format([P.id])')
        rt, ft = _table([cond])
        # the same attributes, under the kind and scope of the one-rule table
        req = {"principal": {k: v for k, v in req["principal"].items() if k != "scope"},
               "resource": dict({k: v for k, v in req["resource"].items() if k != "scope"}, kind="leave_request")}
        sub = tmp_path / str(i)
        sub.mkdir()
        want = _kernel_core(rt, ft, [dict(req, actions=["a0"])], sub)
        assert (want == 1).all(), cond


# ---- differential ----------------------------------------------------------------------------------------------------------
_ATTR_VALUES = [0, 7, -3, 2.5, -0.125, 1e-9, 6.02e23, 1e200, 5e-324, 0.1, 123456.0, 1e6, "x", "", "héllo", 'q"\\\n\t',
                "2021-04-20T10:00:20.5Z", "-1h2m3.25s", True, False, None, [], [1, "a"], [2.5, [True, None]], {"k": 1, "a": "b"}, {"z": [1], "y": {"q": 0}}]
_VERBS = ["%s", "%d", "%f", "%.2f", "%.0f", "%e", "%.3e", "%b", "%x", "%X", "%o", "%.1s"]
_LITS = ["", "id:", "-", "%%", "é", " "]
_ARGS = ["P.attr.a", "P.attr.b", "R.attr.c", "P.id", "1", "-7", "2.5", '"s"', "true", "null", "3u", 'b"hi"', '[1, "a"]', '{"k": 2}',
         "timestamp(R.attr.ts)", "duration(R.attr.d)", "P.attr.a", "R.attr.c"]


def _random_format(rng):
    n = rng.randint(1, 3)
    fmt = "".join(rng.choice(_LITS) + rng.choice(_VERBS) for _ in range(n)) + rng.choice(_LITS)
    if rng.random() < 0.15:
        return f'"{fmt}".format(R.attr.lst)'
    args = ", ".join(rng.choice(_ARGS) for _ in range(n + (rng.random() < 0.1)))
    if rng.random() < 0.1:
        args = ", ".join(rng.choice(_ARGS) for _ in range(max(0, n - 1)))
    return f'"{fmt}".format([{args}])'


def _random_request(rng, i):
    def v():
        return rng.choice(_ATTR_VALUES)
    p = {"a": v(), "b": v()}
    r = {"c": v(), "ts": rng.choice(["2021-04-20T10:00:20.021-05:00", "1999-12-31T23:59:59.999999999Z", "2000-01-01T00:00:00Z", 5]),
         "d": rng.choice(["1h", "-0.5s", "90m0.000001s", "0s", "x"]), "lst": rng.choice([[v(), v()], [v()], [], "nope", [v(), v(), v()]])}
    for d in (p, r):
        for k in list(d):
            if rng.random() < 0.05:
                del d[k]
    return {"principal": {"id": rng.choice(["john", "ann", "é"]), "roles": ["employee"], "attr": p},
            "resource": {"kind": "leave_request", "id": f"r{i}", "attr": r}}


def test_differential_random_format_and_quote(tmp_path):
    """random format / quote conditions x random requests: oracle #1, the interpreter and the generated leaf programs agree"""
    from cerbos_b200.cel.parser import parse
    from oracle.activation import build_activation, build_request
    from oracle.celeval import CelError, eval_expr
    rng = random.Random(20261016)
    compared = 0
    for t in range(8):
        reqs = [_random_request(rng, i) for i in range(200)]
        exprs = []
        while len(exprs) < 32:
            f = _random_format(rng) if rng.random() < 0.85 else rng.choice(['strings.quote(P.attr.a)', 'strings.quote(R.attr.c)', 'strings.quote(P.id)'])
            # compare with the text oracle #1 prints for one of the requests, so that some conditions hold
            r = rng.choice(reqs)
            try:
                val = eval_expr(parse(f), build_activation(build_request(r)), NOW)
            except CelError:
                val = None
            c = f"{f} == {json.dumps(val)}" if isinstance(val, str) else f"size({f}) % 2 == 0"
            exprs += [c, f"!({c})"]
        rt, ft = _table(exprs)
        for r in reqs:
            r["actions"] = [f"a{i}" for i in range(len(exprs))]
        sub = tmp_path / str(t)
        sub.mkdir()
        want = _kernel_core(rt, ft, reqs, sub)
        assert (want == 1).any() and (want == 2).any()
        compared += 2 * want.size
    assert compared >= 50_000


# ---- build time --------------------------------------------------------------------------------------------------------------
def test_a_format_string_that_is_not_a_constant_is_unsupported():
    with pytest.raises(Unsupported, match="format string that is not a constant"):
        _table(['P.attr.dept.format([1]) == "x"'])


def test_a_clause_cut_off_after_its_precision_is_an_error():
    """"%.5" has no verb: the table builder makes every call an error (cel-go reports a malformed clause; oracle #1 has no
    CelError for this text, so the kernel core alone is checked)"""
    rt, ft = _table(['"%.5".format([1]) == "x"', '!("%.5".format([1]) == "x")'])
    b = Encoder(ft.manifest).encode([dict(REQUEST, actions=["a0", "a1"])])
    assert (hostsim.check(ft.blob, b.columns, 1, 2, NOW.ns, mode=1) == 2).all()


def test_list_literal_arguments_reach_the_leaf_program_translator():
    rt, ft = _table(['"id:%s".format([P.id]) == "id:john"'])
    src, _ = hostsim.generate_uc(ft.blob)
    assert "uc_atom_" in src and f"op_fn(c, {hex(L.FNS['FORMAT'])}u" in src and "MKLIST" not in src


def test_nvrtc_unit_of_a_format_table_compiles():
    from cerbos_b200 import capi
    rt, ft = _table(['"id:%s %.2f".format([P.id, P.attr.x]) == "id:john 2.50"', 'strings.quote(P.attr.dept) == "\\"m\\""', 'P.attr.n > 3'])
    n, note = capi.compile_check(ft.blob)
    assert n > 0, note


# ---- the device ----------------------------------------------------------------------------------------------------------
GPU_EXPRS = ['"id:%s".format([P.id]) == "id:" + P.id', '"%.2f".format([P.attr.a]) == "2.50"', '"%s".format([P.attr.a]).startsWith("1")',
             '"%d-%x".format([int(P.attr.i), int(P.attr.i)]) == "255-ff"', 'strings.quote(P.attr.s) == "\\"a\\\\nb\\""', '"%s".format(R.attr.lst) == "[1, x]"',
             '"%e".format([P.attr.a]).endsWith("e+00")', 'P.attr.a > 1.0', 'R.attr.c == "x"', 'P.attr.s in ["a\\nb", "q"]']


def _gpu_requests(n):
    rng = random.Random(7)
    reqs = []
    for i in range(n):
        reqs.append({"principal": {"id": rng.choice(["john", "ann"]), "roles": ["employee"],
                                   "attr": {"a": rng.choice([2.5, 1.25, 10.0, "x", None, 1e21, 0.1]), "i": rng.choice([255, 0, -3]),
                                            "s": rng.choice(["a\nb", "q", 'a"b'])}},
                     "resource": {"kind": "leave_request", "id": f"r{i}", "attr": {"c": rng.choice(["x", "y"]), "lst": rng.choice([[1, "x"], [2], [], "z"])}},
                     "actions": [f"a{k}" for k in range(len(GPU_EXPRS))]})
    return reqs


@pytest.mark.gpu
def test_format_conditions_on_the_device(monkeypatch):
    from cerbos_b200 import capi
    from cerbos_b200 import narrow as NW
    from cerbos_b200.engine import Engine
    rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}} for i, e in enumerate(GPU_EXPRS)]
    pols = [{"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "leave_request", "version": "default", "rules": rules}}]
    reqs = _gpu_requests(3001)
    monkeypatch.setenv("CERBOS_B200_UC", "1")      # the unique-condition kernels also for a table of one block shape
    o = CheckOracle(build_rule_table(pols))
    want = [{a: {1: "EFFECT_ALLOW", 2: "EFFECT_DENY"}.get(v["effect"], v["effect"]) for a, v in o.check(r, NOW)["actions"].items()} for r in reqs]
    bad = dict(reqs[0], principal=dict(reqs[0]["principal"], attr=dict(reqs[0]["principal"]["attr"], a=list(range(1000)))))
    names = {1: "EFFECT_ALLOW", 2: "EFFECT_DENY"}
    for env in ({}, {"CERBOS_B200_NO_JIT": "1"}):
        monkeypatch.delenv("CERBOS_B200_NO_JIT", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng = Engine(pols)
        try:
            specialised, note = eng.table.wait_ready()
            assert specialised == (not env), note
            got = eng.check(reqs, now_ns=NOW.ns)
            assert [{a: v["effect"] for a, v in g["actions"].items()} for g in got] == want, env
            if not env:
                cfg = eng.ctx.last_kernel_config()
                assert cfg["table_specialised"] and cfg["unique_conditions"], cfg
            # a request that must flag fails the whole call: %s of a 1000-element list outgrows the scratch arena
            with pytest.raises(capi.CgpuError) as ei:
                eng.check([bad] + reqs[:5], now_ns=NOW.ns)
            assert ei.value.code == -3      # CGPU_ERR_UNSUPPORTED
            if not env:
                # the narrow wire form of the same batches
                nb = NW.narrow_batch(eng.encoder.encode(reqs), len(eng.encoder.slots))
                eff = eng.table.check_narrow(nb, NOW.ns)
                assert [{f"a{k}": names[int(eff[i, k])] for k in range(len(GPU_EXPRS))} for i in range(len(reqs))] == want
                nb = NW.narrow_batch(eng.encoder.encode([bad] + reqs[:5]), len(eng.encoder.slots))
                with pytest.raises(capi.CgpuError) as ei:
                    eng.table.check_narrow(nb, NOW.ns)
                assert ei.value.code == -3
        finally:
            eng.ctx.close()
