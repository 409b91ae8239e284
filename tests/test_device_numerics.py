"""CEL arithmetic, conversions, ext.Math, number printing and durations on the device, against exact references.

Every expected answer here is computed in this file from the rule cel-go (and the Go library under it) states, with exact
integers, `fractions.Fraction` or Python floats (IEEE binary64, round to nearest even on x86-64).  None comes from one of
the project's evaluators: their agreeing with each other says nothing about cel-go.

The harness: one resource policy per table.  Each condition gets one rule and its negation the next, so a vector's two
effects tell the three outcomes apart: holds (ALLOW, DENY), false (DENY, ALLOW), error (DENY, DENY).  Operands and
expected results travel as request attributes, never as literals (the table builder folds constants): ints and uints as
decimal strings through int() / uint(), doubles as JSON numbers (NaN and +-Inf pass through the encoder), texts as strings.
Double results are compared as `r == e` and as `1.0 / r == 1.0 / e`, which pins the sign of a zero.

Where each family runs:
  * CPU: the host build of the kernel core, interpreter (hostsim mode 1) and generated leaf programs (mode 4), on every
    vector; oracle #1 on a seeded sample;
  * GPU: the general kernel (CERBOS_B200_NO_JIT=1), the NVRTC unique-condition kernel with leaf programs, the metadata
    kernel on a sample, and the narrow wire path for the printing and narrow-column families;
  * the NVRTC unit of a table that multiplies, adds and subtracts doubles is disassembled: no contracted multiply-add.

Out of scope (the device flags them as unsupported): string() of a fractional double, ints above 2^47 inside lists,
timestamps out of the int64-nanosecond range, and duration fractions of more than 9 digits (time.ParseDuration scales
those through float64; DESIGN.md section 6)."""
import functools
import math
import os
import random
import re
import shutil
import struct
import subprocess
from decimal import Decimal
from fractions import Fraction

import numpy as np
import pytest

from cerbos_b200 import narrow as NW
from cerbos_b200.encode import Encoder
from cerbos_b200.policy.compile import build_rule_table
from cerbos_b200.table.flatten import flatten
from hostsim import driver as hostsim
from oracle.celeval import parse_timestamp
from oracle.check import CheckOracle
from test_format import SPECIAL

NOW = parse_timestamp("2021-04-22T10:05:20.021-05:00")
HOLDS, FALSE, ERROR = "holds", "false", "error"
_EFFECTS = {HOLDS: (1, 2), FALSE: (2, 1), ERROR: (2, 2)}
I64_MIN, I64_MAX, U64_MAX = -2 ** 63, 2 ** 63 - 1, 2 ** 64 - 1
INF, NAN = math.inf, math.nan


class _Err:
    def __repr__(self):
        return "ERR"


ERR = _Err()     # the operation is a CEL error


# ---- the harness ----------------------------------------------------------------------------------------------------------
class Probe:
    """One table: up to 16 conditions (32 rules with their negations) and the vectors run through it.
    vectors: [(attributes of the principal, [outcome of each condition])]"""

    def __init__(self, family, conds, vectors):
        assert 0 < len(conds) <= 16 and vectors
        assert all(len(o) == len(conds) for _, o in vectors)
        if len(vectors) % 32 == 0:      # ragged batches only: the last warp is partly empty
            vectors = vectors + [vectors[1 % len(vectors)]]
        self.family, self.conds, self.vectors = family, conds, vectors
        exprs = [e for c in conds for e in (c, f"!({c})")]
        rules = [{"actions": [f"a{i}"], "effect": "EFFECT_ALLOW", "roles": ["*"], "condition": {"match": {"expr": e}}} for i, e in enumerate(exprs)]
        pol = {"apiVersion": "api.cerbos.dev/v1", "resourcePolicy": {"resource": "leave_request", "version": "default", "rules": rules}}
        self.rt = build_rule_table([pol])
        self.ft = flatten(self.rt)
        self.k = len(exprs)

    def request(self, i):
        return {"principal": {"id": "p", "roles": ["employee"], "attr": self.vectors[i][0]},
                "resource": {"kind": "leave_request", "id": f"r{i}", "attr": {}}, "actions": [f"a{j}" for j in range(self.k)]}

    def want(self, idx=None):
        idx = range(len(self.vectors)) if idx is None else idx
        return np.array([[e for o in self.vectors[i][1] for e in _EFFECTS[o]] for i in idx], dtype=np.uint8)

    @functools.cached_property
    def batch(self):
        return Encoder(self.ft.manifest).encode([self.request(i) for i in range(len(self.vectors))])

    def outcomes(self):
        return {o for _, os_ in self.vectors for o in os_}


def _eq(r, e):
    """outcome of `<op> == <expected>`: r the exact result of the operation (ERR: a CEL error), e the expected value"""
    return ERROR if r is ERR else HOLDS if r == e else FALSE


def _fdiv(x, y):
    """IEEE division (Python raises on a zero divisor): x / +-0 is +-Inf with the product of the signs, 0 / 0 and NaN / 0 NaN"""
    if y == 0:
        if x == 0 or x != x:
            return NAN
        return math.copysign(INF, x) * math.copysign(1.0, y)
    return x / y


def _dbl_forms(r, e):
    """outcomes of `<op> == e` and `1.0 / (<op>) == 1.0 / e` for a double result r (NaN is unequal to everything)"""
    if r is ERR:
        return [ERROR, ERROR]
    return [HOLDS if r == e else FALSE, HOLDS if _fdiv(1.0, r) == _fdiv(1.0, e) else FALSE]


def _wrong_int(r, k, every=5):
    """the expected value of vector k: the exact result, except on every `every`-th vector, where the lowest bit is flipped
    (a false outcome; flipping bit 0 keeps the value in the int64 / uint64 range)"""
    return r ^ 1 if k % every == every // 2 else r


def _wrong_dbl(r, k, every=7):
    return math.nextafter(r, INF) if k % every == every // 2 and math.isfinite(r) else r


# ---- exact references ---------------------------------------------------------------------------------------------------
def _i64(x):
    return x if I64_MIN <= x <= I64_MAX else ERR


def _u64(x):
    return x if 0 <= x <= U64_MAX else ERR


def _tdiv(a, b):
    """Go's integer division: the quotient truncated toward zero"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


# cel-go common/types/int.go: Add / Subtract / Multiply / Negate overflow int64 -> "integer overflow" (addInt64Checked ...);
# Divide: a zero divisor -> "divide by zero", MinInt64 / -1 -> overflow; Go's `/` truncates toward zero.  Modulo: a zero
# divisor -> "modulus by zero", MinInt64 % -1 -> overflow (moduloInt64Checked); Go's `%` takes the dividend's sign.
# ext.Math abs: MinInt64 has no int64 absolute value -> overflow.
INT_OPS = [("add", "+", lambda a, b: _i64(a + b)), ("sub", "-", lambda a, b: _i64(a - b)), ("mul", "*", lambda a, b: _i64(a * b)),
           ("div", "/", lambda a, b: ERR if b == 0 else _i64(_tdiv(a, b))),
           ("mod", "%", lambda a, b: ERR if b == 0 or (a == I64_MIN and b == -1) else a - b * _tdiv(a, b))]
INT_UNARY = [("neg", "-int(P.attr.a)", lambda a: _i64(-a)), ("abs", "math.abs(int(P.attr.a))", lambda a: _i64(abs(a)))]
# cel-go common/types/uint.go: Add / Multiply wrap -> "unsigned integer overflow", Subtract below 0 -> overflow; Divide / Modulo
# by zero -> error.
UINT_OPS = [("add", "+", lambda a, b: _u64(a + b)), ("sub", "-", lambda a, b: _u64(a - b)), ("mul", "*", lambda a, b: _u64(a * b)),
            ("div", "/", lambda a, b: ERR if b == 0 else a // b), ("mod", "%", lambda a, b: ERR if b == 0 else a % b)]


def _int_of_double(d):
    """cel-go Double.ConvertToType(IntType), doubleToInt64Checked: NaN, +-Inf, d <= float64(MinInt64) = -2^63 and
    d >= float64(MaxInt64) = 2^63 are "integer overflow"; anything else truncates toward zero"""
    return ERR if not math.isfinite(d) or d <= -2.0 ** 63 or d >= 2.0 ** 63 else int(d)


def _uint_of_double(d):
    """doubleToUint64Checked: NaN, +-Inf, d < 0 and d >= 2^64 are errors (so uint(-0.5) fails and uint(-0.0) is 0)"""
    return ERR if not math.isfinite(d) or d < 0 or d >= 2.0 ** 64 else int(d)


def _parse_int(s):
    """String.ConvertToType(IntType) is strconv.ParseInt(s, 10, 64): one optional sign, then ASCII digits only (base 10:
    no prefix, no underscores), in range"""
    return _i64(int(s)) if re.fullmatch(r"[+-]?[0-9]+", s) else ERR


def _parse_uint(s):
    """String.ConvertToType(UintType) is strconv.ParseUint(s, 10, 64): "A sign prefix is not permitted"; ASCII digits, in range"""
    return _u64(int(s)) if re.fullmatch(r"[0-9]+", s) else ERR


def _cmp(x, y):
    return (x > y) - (x < y)


def _cmp_double_int(d, i):
    """cel-go common/types/compare.go compareDoubleInt: a range test first (d < MinInt64, d > MaxInt64, both as float64),
    then the two compared as doubles, the int rounded to the nearest double: lossy on purpose"""
    if d < -2.0 ** 63:
        return -1
    if d > 2.0 ** 63:
        return 1
    return _cmp(d, float(i))


def _cmp_double_uint(d, u):
    """compareDoubleUint: d < 0 -> -1, d > float64(MaxUint64) = 2^64 -> 1, else as doubles"""
    if d < 0:
        return -1
    if d > 2.0 ** 64:
        return 1
    return _cmp(d, float(u))


def _rel(op, c):
    """outcome of `x <op> y` from their comparison c (None: a NaN operand).  With a NaN, == is false and != true; ordering
    it is cel-go's "NaN values cannot be ordered" error"""
    if c is None:
        return {"==": FALSE, "!=": HOLDS}.get(op, ERROR)
    return HOLDS if {"==": c == 0, "!=": c != 0, "<": c < 0, "<=": c <= 0, ">": c > 0, ">=": c >= 0}[op] else FALSE


def _signed_zero(r, x):
    return math.copysign(0.0, x) if r == 0 else r


def _go_round(x):
    """Go math.Round: half away from zero, exactly (floor(|x| + 0.5) in doubles would round 0.49999999999999994 up)"""
    if not math.isfinite(x) or x == 0:
        return x
    return math.copysign(float(math.floor(abs(Fraction(x)) + Fraction(1, 2))), x)


# Go math.Ceil / Floor / Trunc keep +-0, +-Inf and NaN, and a zero result takes the sign of the argument (Ceil(-0.5) = -0)
def _go_ceil(x):
    return x if not math.isfinite(x) or x == 0 else _signed_zero(float(math.ceil(x)), x)


def _go_floor(x):
    return x if not math.isfinite(x) or x == 0 else _signed_zero(float(math.floor(x)), x)


def _go_trunc(x):
    return x if not math.isfinite(x) or x == 0 else _signed_zero(float(math.trunc(x)), x)


def _go_sqrt(x):
    """Go math.Sqrt, IEEE sqrt (correctly rounded; Sqrt(-0) = -0, a negative number NaN).  ext.Math sqrt of an int / uint is
    math.Sqrt(float64(v)): the integer rounded to the nearest double first"""
    return NAN if x < 0 else math.sqrt(x)


def _sign_d(x):
    """ext.Math sign of a double: NaN stays NaN, otherwise -1.0 / 0.0 / 1.0 (compared by value: the sign of a zero result
    is not pinned here)"""
    return x if x != x else float(_cmp(x, 0.0))


def _shl(x, k, bits_signed):
    """ext.Math bitShiftLeft: a negative count is an error, a count of 64 or more gives 0 (Go's shift semantics)"""
    if k < 0:
        return ERR
    r = (x << k) & U64_MAX if k < 64 else 0
    return r - 2 ** 64 if bits_signed and r > I64_MAX else r


def _shr(x, k, bits_signed):
    """ext.Math bitShiftRight: on an int the shift is logical (the bits are shifted as a uint64)"""
    if k < 0:
        return ERR
    r = (x & U64_MAX) >> k if k < 64 else 0
    return r - 2 ** 64 if bits_signed and r > I64_MAX else r


def _fmt_g(d):
    """%s of a double is strconv.FormatFloat(d, 'g', -1, 64): the shortest digits that round-trip (Python's repr gives the
    same, correctly rounded), in exponent form when the decimal exponent is below -4 or at least 6 (strconv/ftoa.go: the
    shortest form sets eprec = 6), with at least two exponent digits.  NaN and +-Inf print as NaN, Infinity, -Infinity."""
    if d != d:
        return "NaN"
    if math.isinf(d):
        return "Infinity" if d > 0 else "-Infinity"
    sign = "-" if math.copysign(1.0, d) < 0 else ""
    if d == 0:
        return sign + "0"
    t = Decimal(repr(abs(d))).normalize().as_tuple()      # the digits without trailing zeros
    digits = "".join(map(str, t.digits))
    dp = len(digits) + t.exponent          # the decimal point sits after digit dp (dp <= 0: before leading zeros)
    x = dp - 1
    if x < -4 or x >= 6:
        m = digits[0] + ("." + digits[1:] if len(digits) > 1 else "")
        return f"{sign}{m}e{'-' if x < 0 else '+'}{abs(x):02d}"
    if dp <= 0:
        return f"{sign}0.{'0' * -dp}{digits}"
    if dp >= len(digits):
        return sign + digits + "0" * (dp - len(digits))
    return f"{sign}{digits[:dp]}.{digits[dp:]}"


def _fmt_fe(d, p, verb):
    """%.{p}f / %.{p}e: the exact decimal value rounded once, ties to even (Python's formatting is exact); NaN and +-Inf
    print as NaN, Infinity, -Infinity under every verb (cel-go ext/strings.go formatting of doubles)"""
    if not math.isfinite(d):
        return _fmt_g(d)
    return format(d, f".{p}{verb}")


# Go time.ParseDuration (time/format.go), which cel-go's duration(string) calls: [+-], then "0" alone or one or more
# <digits>[.<digits>]<unit>; units ns us (U+00B5)s (U+03BC)s ms s m h.  The whole part overflows above 2^63; the fraction is
# added as uint64(float64(f) * (float64(unit) / scale)); the total may reach 2^63 only with a minus sign.
_UNITS = {"ns": 1, "us": 1000, "µs": 1000, "μs": 1000, "ms": 10 ** 6, "s": 10 ** 9, "m": 60 * 10 ** 9, "h": 3600 * 10 ** 9}


def _go_parse_duration(s):
    neg = False
    if s and s[0] in "+-":
        neg, s = s[0] == "-", s[1:]
    if s == "0":
        return 0
    if not s:
        return ERR
    d = 0
    while s:
        if not (s[0] == "." or s[0].isascii() and s[0].isdigit()):
            return ERR
        m = re.match(r"[0-9]*", s)
        pre, s = m.group(), s[m.end():]
        v = int(pre) if pre else 0
        if v > 2 ** 63:
            return ERR
        f, scale, post = 0, 1.0, False
        if s.startswith("."):
            m = re.match(r"[0-9]*", s[1:])
            frac, s, post = m.group(), s[1 + m.end():], bool(m.group())
            assert len(frac) <= 18        # (leadingFraction drops digits past int64 precision; not generated here)
            f, scale = (int(frac), 10.0 ** len(frac)) if frac else (0, 1.0)
        if not pre and not post:
            return ERR
        m = re.match(r"[^0-9.]*", s)
        u, s = m.group(), s[m.end():]
        if u not in _UNITS:
            return ERR
        unit = _UNITS[u]
        if v > 2 ** 63 // unit:
            return ERR
        v *= unit
        if f > 0:
            v += int(float(f) * (float(unit) / scale))
            if v > 2 ** 63:
                return ERR
        d += v
        if d > 2 ** 63:
            return ERR
    if neg:
        return -d
    return d if d <= I64_MAX else ERR


# ---- families -------------------------------------------------------------------------------------------------------------
INT_EDGES = sorted({0, 1, -1, 2, -2, 3, -3, 7, -7, 10, -10, 2 ** 31 - 1, -(2 ** 31 - 1), 2 ** 31, -2 ** 31, 2 ** 31 + 1, -(2 ** 31 + 1),
                    2 ** 32, -2 ** 32, 2 ** 32 + 1, -(2 ** 32 + 1), 3037000499, -3037000499, 3037000500, -3037000500, 2 ** 53 + 1, -(2 ** 53 + 1),
                    2 ** 62, -2 ** 62, 2 ** 62 + 1, -(2 ** 62 + 1), I64_MAX, I64_MAX - 1, I64_MIN, I64_MIN + 1, 6148914691236517205, -6148914691236517206})
UINT_EDGES = sorted({0, 1, 2, 3, 7, 10, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 4294967295, 4294967296, 4294967297,
                     2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 62, 2 ** 63 - 1, 2 ** 63, 2 ** 63 + 1, U64_MAX - 1, U64_MAX, 6074001000, 12297829382473034410,
                     3037000499, 3037000500, 2 ** 48 + 3, 10 ** 19, 10 ** 19 + 1})


def _product_boundaries(limit, signed):
    """for b across every magnitude (both signs when signed): a = floor(limit / b) and a + 1, the last product in range and
    the first out of it"""
    out = []
    bs = sorted({2 ** e + d for e in range(1, 64) for d in (-1, 0, 1)} | {3, 5, 7, 10, 3037000499, 3037000500, 4294967295, 10 ** 9, 10 ** 18})
    for b in bs:
        for s in ((1, -1) if signed else (1,)):
            bb = s * b
            if signed and not I64_MIN <= bb <= I64_MAX or not signed and bb > U64_MAX:
                continue
            a = limit // bb
            for x in (a, a + 1, -a, -a - 1) if signed else (a, a + 1):
                if (I64_MIN <= x <= I64_MAX) if signed else (0 <= x <= U64_MAX):
                    out += [(x, bb), (bb, x)]
    return out


def _int_family():
    pairs = list(dict.fromkeys([(a, b) for a in INT_EDGES for b in INT_EDGES] + _product_boundaries(I64_MAX, True) + _product_boundaries(-I64_MIN, True)))
    conds = [f"int(P.attr.a) {sym} int(P.attr.b) == int(P.attr.{name})" for name, sym, _ in INT_OPS] + \
            [f"{expr} == int(P.attr.{name})" for name, expr, _ in INT_UNARY]
    vecs = []
    for k, (a, b) in enumerate(pairs):
        attrs, outs = {"a": str(a), "b": str(b)}, []
        for name, r in [(n, f(a, b)) for n, _, f in INT_OPS] + [(n, f(a)) for n, _, f in INT_UNARY]:
            e = 0 if r is ERR else _wrong_int(r, k)
            attrs[name] = str(e)
            outs.append(_eq(r, e))
        vecs.append((attrs, outs))
    return [Probe("int64", conds, vecs)]


def _uint_family():
    pairs = list(dict.fromkeys([(a, b) for a in UINT_EDGES for b in UINT_EDGES] + _product_boundaries(U64_MAX, False)))
    conds = [f"uint(P.attr.a) {sym} uint(P.attr.b) == uint(P.attr.{name})" for name, sym, _ in UINT_OPS]
    vecs = []
    for k, (a, b) in enumerate(pairs):
        attrs, outs = {"a": str(a), "b": str(b)}, []
        for name, _, f in UINT_OPS:
            r = f(a, b)
            e = 0 if r is ERR else _wrong_int(r, k)
            attrs[name] = str(e)
            outs.append(_eq(r, e))
        vecs.append((attrs, outs))
    return [Probe("uint64", conds, vecs)]


DBL_SPECIAL = [0.0, -0.0, 1.0, -1.5, 3.0, 0.1, 5e-324, -5e-324, 2.2250738585072014e-308, -2.225073858507201e-308, 1e-300, 1e308,
               -1.7976931348623157e308, INF, -INF, NAN]


def _fma_sensitive(n, seed):
    """n triples (a, b, c) whose fused a*b + c (one rounding, exact via Fraction) differs from round(round(a*b) + c)"""
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        a = rng.uniform(1, 2) * 2.0 ** rng.randint(-80, 80) * rng.choice((1, -1))
        b = rng.uniform(1, 2) * 2.0 ** rng.randint(-80, 80) * rng.choice((1, -1))
        p = a * b
        m = rng.randrange(4)
        c = -p if m == 0 else -p * (1 + rng.randint(-64, 64) * 2.0 ** -52) if m == 1 else \
            rng.uniform(-1, 1) * abs(p) * 2.0 ** rng.randint(-40, 2) if m == 2 else -p + rng.uniform(-1, 1) * abs(p) * 2.0 ** -50
        fused = float(Fraction(a) * Fraction(b) + Fraction(c))     # int / int true division: correctly rounded
        two = p + c
        if fused != two or math.copysign(1.0, fused) != math.copysign(1.0, two):
            out.append((a, b, c))
    return out


# a*b + c, a*b - n (n = -c) and c + a*b: the same fused value, three ways of writing the unfused one
FMA_OPS = [("r1", "P.attr.a * P.attr.b + P.attr.c", lambda a, b, c: a * b + c), ("r2", "P.attr.a * P.attr.b - P.attr.n", lambda a, b, c: a * b - -c),
           ("r3", "P.attr.c + P.attr.a * P.attr.b", lambda a, b, c: c + a * b)]
DBL_OPS = [("s", "P.attr.a + P.attr.b", lambda a, b, c: a + b), ("d", "P.attr.a - P.attr.b", lambda a, b, c: a - b),
           ("m", "P.attr.a * P.attr.b", lambda a, b, c: a * b), ("q", "P.attr.a / P.attr.b", lambda a, b, c: _fdiv(a, b))]


def _double_family():
    """each operation rounded once to nearest even; division by zero is +-Inf or NaN, not an error; subnormals are kept"""
    triples = _fma_sensitive(16384, 3) + [(a, b, c) for a in DBL_SPECIAL for b in DBL_SPECIAL for c in DBL_SPECIAL[::3]]
    ops = FMA_OPS + DBL_OPS
    vecs = []
    for k, (a, b, c) in enumerate(triples):
        attrs = {"a": a, "b": b, "c": c, "n": -c}
        res = {}
        for name, _, f in ops:
            r = f(a, b, c)
            attrs[name] = _wrong_dbl(r, k)
            res[name] = r
        vecs.append((attrs, res))
    probes = []
    for group in (FMA_OPS, DBL_OPS):
        conds, outs_of = [], []
        for name, expr, _ in group:
            conds += [f"{expr} == P.attr.{name}", f"1.0 / ({expr}) == 1.0 / P.attr.{name}", f"math.isNaN({expr}) == math.isNaN(P.attr.{name})"]
        pv = []
        for attrs, res in vecs:
            o = []
            for name, _, _ in group:
                o += _dbl_forms(res[name], attrs[name]) + [HOLDS if math.isnan(res[name]) == math.isnan(attrs[name]) else FALSE]
            pv.append((attrs, o))
        probes.append(Probe("double", conds, pv))
    return probes


def _near(x):
    return [math.nextafter(x, -INF), x, math.nextafter(x, INF)]


CONV_DOUBLES = sorted({y for x in (2.0 ** 53, 2.0 ** 63, 2.0 ** 64, 2.0 ** 52, 2.0 ** 32, 1.0, 0.5) for s in (1, -1) for y in _near(s * x)}
                      | {-0.0, 1.5, -1.5, 2.5, 9007199254740993.0, 1e300, -1e300, 5e-324}) + [-0.0, NAN, INF, -INF]
CONV_INTS = [0, 1, -1, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, 2 ** 53 + 3, -(2 ** 53 + 1), I64_MAX, I64_MAX - 511, I64_MAX - 512, I64_MAX - 1024,
             I64_MIN, I64_MIN + 1, 2 ** 62, 9007199254740993, -2]
CONV_UINTS = [0, 1, 2 ** 53 + 1, 2 ** 63 - 1, 2 ** 63, 2 ** 63 + 1, 2 ** 63 + 1024, 2 ** 63 + 1025, U64_MAX, U64_MAX - 1024, U64_MAX - 1025, U64_MAX - 2048, 2 ** 53, 7]
CONV_TEXTS = ["0", "5", "+5", "-5", "+0", "-0", "007", "9223372036854775807", "9223372036854775808", "-9223372036854775808", "-9223372036854775809",
              "18446744073709551615", "18446744073709551616", "+18446744073709551615", "", "+", "-", " 1", "1 ", "1_000", "0x10", "1e3", "1.0",
              "٣", "99999999999999999999999", "00000000000000000000000000001", "--1", "+-1"]


def _conversion_family():
    vecs = []
    n = max(len(CONV_DOUBLES), len(CONV_INTS), len(CONV_UINTS), len(CONV_TEXTS)) * 3
    for k in range(n):
        d, i, u, s = CONV_DOUBLES[k % len(CONV_DOUBLES)], CONV_INTS[(7 * k) % len(CONV_INTS)], CONV_UINTS[(5 * k) % len(CONV_UINTS)], CONV_TEXTS[k % len(CONV_TEXTS)]
        res = [("di", _int_of_double(d), "int"), ("du", _uint_of_double(d), "uint"), ("id", float(i), None), ("ud", float(u), None),
               ("ui", _i64(u), "int"), ("iu", _u64(i), "uint"), ("si", _parse_int(s), "int"), ("su", _parse_uint(s), "uint")]
        attrs, outs = {"d": d, "i": str(i), "u": str(u), "s": s}, []
        for name, r, kind in res:
            if kind:
                e = 0 if r is ERR else _wrong_int(r, k, 7)
                attrs[name] = str(e)
            else:                        # double(int) / double(uint): Go's float64(v) rounds to nearest even, as Python's float(v)
                e = attrs[name] = _wrong_dbl(r, k)
            outs.append(_eq(r, e))
        vecs.append((attrs, outs))
    conds = ["int(P.attr.d) == int(P.attr.di)", "uint(P.attr.d) == uint(P.attr.du)", "double(int(P.attr.i)) == P.attr.id",
             "double(uint(P.attr.u)) == P.attr.ud", "int(uint(P.attr.u)) == int(P.attr.ui)", "uint(int(P.attr.i)) == uint(P.attr.iu)",
             "int(P.attr.s) == int(P.attr.si)", "uint(P.attr.s) == uint(P.attr.su)"]
    # cross-type ordering and equality: double against int (double on the left), uint against double (uint on the left),
    # int against uint (exact)
    ops = ["==", "!=", "<", "<=", ">", ">="]
    cconds = [f"P.attr.d {op} int(P.attr.i)" for op in ops] + [f"uint(P.attr.u) {op} P.attr.d" for op in ops] + \
             [f"int(P.attr.i) {op} uint(P.attr.u)" for op in ("<", "==", ">=")]
    cvecs = []
    for k, (d, i) in enumerate((d, i) for d in CONV_DOUBLES for i in CONV_INTS):
        u = CONV_UINTS[k % len(CONV_UINTS)]
        cd = None if d != d else _cmp_double_int(d, i)
        cu = None if d != d else -_cmp_double_uint(d, u)
        outs = [_rel(op, cd) for op in ops] + [_rel(op, cu) for op in ops] + [_rel(op, _cmp(i, u)) for op in ("<", "==", ">=")]
        cvecs.append(({"d": d, "i": str(i), "u": str(u)}, outs))
    return [Probe("conversions", conds, vecs), Probe("conversions", cconds, cvecs)]


MATH_DOUBLES = [0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 3.5, -3.5, 2.0 ** 52 - 0.5, -(2.0 ** 52 - 0.5), 2.0 ** 51 + 0.5, -(2.0 ** 51 + 0.5), 2.0 ** 53 - 1,
                2.0 ** 53, 2.0 ** 52 + 1, 0.49999999999999994, -0.49999999999999994, 0.5000000000000001, -0.9999999999999999, 0.0, -0.0, 5e-324, -5e-324,
                2.2250738585072014e-308, -1e-310, 1e300, -1e300, 1.7976931348623157e308, INF, -INF, NAN, 4.0, 2.0, 0.1, -0.1, 1e-5, 123456.789]
MATH_FNS = [("round", "math.round", _go_round), ("ceil", "math.ceil", _go_ceil), ("floor", "math.floor", _go_floor),
            ("trunc", "math.trunc", _go_trunc), ("abs", "math.abs", math.fabs), ("sqrt", "math.sqrt", _go_sqrt)]


def _math_family():
    rng = random.Random(5)
    xs = MATH_DOUBLES + [rng.randint(-2 ** 40, 2 ** 40) + 0.5 for _ in range(500)] + \
        [struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0] for _ in range(1500)] + [rng.uniform(0, 1e6) for _ in range(500)]
    xs = list({repr(x): x for x in xs}.values())
    vecs = []
    for k, x in enumerate(xs):
        res = {name: f(x) for name, _, f in MATH_FNS}
        res["sign"] = _sign_d(x)
        vecs.append(({"x": x, **{n: _wrong_dbl(r, k) for n, r in res.items()}}, res))
    conds, nconds = [], []
    for name, fn, _ in MATH_FNS:
        conds += [f"{fn}(P.attr.x) == P.attr.{name}", f"1.0 / {fn}(P.attr.x) == 1.0 / P.attr.{name}"]
        nconds.append(f"math.isNaN({fn}(P.attr.x)) == math.isNaN(P.attr.{name})")
    conds.append("math.sign(P.attr.x) == P.attr.sign")
    nconds.append("math.isNaN(math.sign(P.attr.x)) == math.isNaN(P.attr.sign)")
    p1 = [(a, [o for n, _, _ in MATH_FNS for o in _dbl_forms(r[n], a[n])] + [_eq(r["sign"], a["sign"])]) for a, r in vecs]
    p2 = [(a, [HOLDS if math.isnan(r[n]) == math.isnan(a[n]) else FALSE for n in [m for m, _, _ in MATH_FNS] + ["sign"]]) for a, r in vecs]
    # integers: shifts by 0, 1, 31, 63, 64, 65 and -1; sqrt of an int / uint (converted to double first); sign and abs
    ivecs = []
    ks = [0, 1, 31, 63, 64, 65, -1, 1000]
    for k, (i, sh) in enumerate((i, sh) for i in INT_EDGES for sh in ks):
        u = UINT_EDGES[k % len(UINT_EDGES)]
        res = [("shl", _shl(i, sh, True), "int"), ("shr", _shr(i, sh, True), "int"), ("ushl", _shl(u, sh, False), "uint"),
               ("ushr", _shr(u, sh, False), "uint"), ("isign", _cmp(i, 0), "int"), ("iabs", _i64(abs(i)), "int"),
               ("isqrt", _go_sqrt(float(i)), None), ("usqrt", _go_sqrt(float(u)), None)]
        attrs, outs = {"i": str(i), "u": str(u), "k": str(sh)}, []
        for name, r, kind in res:
            if kind:
                e = 0 if r is ERR else _wrong_int(r, k, 7)
                attrs[name] = str(e)
            else:
                e = attrs[name] = _wrong_dbl(r, k)
            outs.append(_eq(r, e))
        ivecs.append((attrs, outs))
    iconds = ["math.bitShiftLeft(int(P.attr.i), int(P.attr.k)) == int(P.attr.shl)", "math.bitShiftRight(int(P.attr.i), int(P.attr.k)) == int(P.attr.shr)",
              "math.bitShiftLeft(uint(P.attr.u), int(P.attr.k)) == uint(P.attr.ushl)", "math.bitShiftRight(uint(P.attr.u), int(P.attr.k)) == uint(P.attr.ushr)",
              "math.sign(int(P.attr.i)) == int(P.attr.isign)", "math.abs(int(P.attr.i)) == int(P.attr.iabs)",
              "math.sqrt(int(P.attr.i)) == P.attr.isqrt", "math.sqrt(uint(P.attr.u)) == P.attr.usqrt"]
    return [Probe("math", conds, p1), Probe("math", nconds, p2), Probe("math", iconds, ivecs)]


PRECISIONS = (0, 1, 2, 6, 17, 20)


def _print_doubles():
    rng = np.random.default_rng(11)
    bits = rng.integers(0, 2 ** 64, size=30000, dtype=np.uint64)
    rnd = bits.view(np.float64)
    xs = [float(x) for x in rnd[np.isfinite(rnd)]]
    xs += [math.ldexp(1.0, e) for e in range(-1074, 1024)]                  # every power of two
    xs += [10.0 ** k for k in range(-30, 31)] + [float(f"1e{k}") for k in range(-30, 31)] + list(SPECIAL) + [NAN, INF, -INF]
    r = random.Random(12)                                                   # halfway cases of %.{p}f: n + odd / 2^m
    xs += [r.choice((1, -1)) * (r.randint(0, 10 ** 6) + r.randrange(1, 2 ** m, 2) / 2 ** m) for m in range(1, 8) for _ in range(150)]
    return list({repr(x): x for x in xs}.values())


def _printing_family():
    xs = _print_doubles()
    verbs = [("g", "%s", lambda d: _fmt_g(d))] + [(f"f{p}", f"%.{p}f", functools.partial(_fmt_fe, p=p, verb="f")) for p in PRECISIONS] + \
            [(f"e{p}", f"%.{p}e", functools.partial(_fmt_fe, p=p, verb="e")) for p in PRECISIONS]
    conds = [f'"{v}".format([P.attr.x]) == P.attr.{name}' for name, v, _ in verbs]
    vecs = []
    for k, x in enumerate(xs):
        attrs, outs = {"x": x}, []
        for name, _, f in verbs:
            t = f(x)
            attrs[name] = t + "0" if k % 11 == 5 else t
            outs.append(HOLDS if attrs[name] == t else FALSE)
        vecs.append((attrs, outs))
    # %d %x %X %o %b of the int64 and uint64 edge sets, and of texts that are not int64 / uint64 (an error)
    ivs = []
    texts = [str(v) for v in INT_EDGES] + [str(v) for v in UINT_EDGES] + ["9223372036854775808", "-9223372036854775809", "18446744073709551616"]
    iverbs = [("d", "d"), ("x", "x"), ("X", "X"), ("o", "o"), ("b", "b")]
    for k, s in enumerate(texts * 3):
        i, u = _parse_int(s), _parse_uint(s)
        attrs, outs = {"s": s}, []
        for kind, v in (("i", i), ("u", u)):
            for name, verb in iverbs:
                t = "" if v is ERR else format(v, verb)
                attrs[kind + name] = t + "1" if k % 5 == 2 else t
                outs.append(ERROR if v is ERR else HOLDS if attrs[kind + name] == t else FALSE)
        ivs.append((attrs, outs))
    iconds = [f'"%{verb}".format([int(P.attr.s)]) == P.attr.i{name}' for name, verb in iverbs] + \
             [f'"%{verb}".format([uint(P.attr.s)]) == P.attr.u{name}' for name, verb in iverbs]
    return [Probe("printing", conds, vecs), Probe("printing", iconds, ivs)]


def _f32(b):
    return float(np.array([b], dtype=np.uint32).view(np.float32)[0])


def _narrow_family():
    """a column of float32-exact doubles and one of small non-negative integers, each printed with %s"""
    rng = random.Random(13)
    xs = [_f32(rng.getrandbits(32) & 0x7FFFFFFF | rng.getrandbits(1) << 31) for _ in range(3000)]
    xs = [x for x in xs if math.isfinite(x)]
    xs += [_f32(m | s << 31) for m in [1, 2, 3, 0x7FFFFF, 0x400000, 0x12345] + [rng.randrange(1, 2 ** 23) for _ in range(200)] for s in (0, 1)]   # subnormals
    xs += [-0.0, 0.0, INF, -INF, NAN, 2.0 ** 24 + 2, 2.0 ** 24, 2.0 ** 24 - 1, 3.4028234663852886e38, 2.0 ** -126, _f32(0x3DCCCCCD), 0.5, 240.0, 255.0]
    vecs = []
    for k, x in enumerate(xs):
        n = k % 240
        s, t = _fmt_g(x), _fmt_g(float(n))
        attrs = {"x": x, "n": n, "s": s + " " if k % 9 == 4 else s, "t": t + " " if k % 9 == 7 else t}
        vecs.append((attrs, [HOLDS if attrs["s"] == s else FALSE, HOLDS if attrs["t"] == t else FALSE]))
    return [Probe("narrow", ['"%s".format([P.attr.x]) == P.attr.s', '"%s".format([P.attr.n]) == P.attr.t'], vecs)]


def _duration_texts():
    rng = random.Random(17)
    out = []
    for u in _UNITS:
        for nd in range(1, 10):
            for whole in ("0", "1", "7", "59", "1234", ""):
                frac = "".join(rng.choice("0123456789") for _ in range(nd))
                out.append(f"{rng.choice(['', '-', '+'])}{whole}.{frac}{u}")
            out += [f"{w}.{'9' * nd}{u}" for w in ("0", "2562047")] + [f"-.{'0' * (nd - 1)}5{u}", f"1.{'0' * (nd - 1)}1{u}"]
    out += ["0", "-0", "+0", "1h30m0.5s", "1.5h1.5m1.5s1.5ms1.5us1.5ns", "2562047h47m16.854775807s", "-2562047h47m16.854775808s",
            "2562047h47m16.854775808s", "2562048h", "9223372036854775807ns", "9223372036854775808ns", "-9223372036854775808ns",
            "1.5", "", "s", ".s", "1.s", "1x", "1hx", "-", "1e3s", "0.000000001s", "153722867m16.854775807s"]
    return out


def _duration_family():
    texts = _duration_texts()
    others = ["0", "1ns", "-1ns", "2562047h47m16.854775807s", "-2562047h47m16.854775808s", "1.5h", "-0.000000001s"]
    vecs = []
    for k, s in enumerate(texts):
        t = others[k % len(others)]
        ds, dt = _go_parse_duration(s), _go_parse_duration(t)
        # cel-go: duration + duration and duration - duration overflow int64 nanoseconds -> error; int(duration) is the
        # nanosecond count
        res = [ds, ERR if ds is ERR or dt is ERR else _i64(ds + dt), ERR if ds is ERR or dt is ERR else _i64(ds - dt)]
        attrs, outs = {"s": s, "t": t}, []
        for name, r in zip(("ns", "sum", "diff"), res):
            e = 0 if r is ERR else _wrong_int(r, k, 7)
            attrs[name] = str(e)
            outs.append(_eq(r, e))
        vecs.append((attrs, outs))
    conds = ["int(duration(P.attr.s)) == int(P.attr.ns)", "int(duration(P.attr.s) + duration(P.attr.t)) == int(P.attr.sum)",
             "int(duration(P.attr.s) - duration(P.attr.t)) == int(P.attr.diff)"]
    return [Probe("duration", conds, vecs)]


FAMILIES = {"int64": _int_family, "uint64": _uint_family, "double": _double_family, "conversions": _conversion_family,
            "math": _math_family, "printing": _printing_family, "narrow": _narrow_family, "duration": _duration_family}
# least number of vectors per family, and the outcome classes each must show
MIN_VECTORS = {"int64": 1600, "uint64": 1000, "double": 16384 + 1000, "conversions": 1000, "math": 2500, "printing": 32768 + 200,
               "narrow": 3000, "duration": 500}
CLASSES = {"int64": {HOLDS, FALSE, ERROR}, "uint64": {HOLDS, FALSE, ERROR}, "double": {HOLDS, FALSE}, "conversions": {HOLDS, FALSE, ERROR},
           "math": {HOLDS, FALSE, ERROR}, "printing": {HOLDS, FALSE, ERROR}, "narrow": {HOLDS, FALSE}, "duration": {HOLDS, FALSE, ERROR}}


@functools.lru_cache(maxsize=None)
def family(name):
    return FAMILIES[name]()


# ---- CPU --------------------------------------------------------------------------------------------------------------------
def test_references_on_written_out_cases():
    """the exact references on cases whose answers cel-go's documentation or the Go library spell out"""
    assert _tdiv(-7, 2) == -3 and -7 - 2 * _tdiv(-7, 2) == -1 and INT_OPS[4][2](7, -2) == 1
    assert INT_OPS[3][2](I64_MIN, -1) is ERR and INT_OPS[4][2](I64_MIN, -1) is ERR and INT_UNARY[0][2](I64_MIN) is ERR
    assert UINT_OPS[1][2](0, 1) is ERR and UINT_OPS[2][2](2 ** 32, 2 ** 32) is ERR
    assert _uint_of_double(-0.5) is ERR and _uint_of_double(-0.0) == 0 and _int_of_double(-2.0 ** 63) is ERR and _int_of_double(2.0 ** 63) is ERR
    assert _int_of_double(math.nextafter(-2.0 ** 63, 0)) == -2 ** 63 + 1024
    assert _parse_uint("+5") is ERR and _parse_int("+5") == 5 and _parse_int("-0") == 0 and _parse_int("1_000") is ERR and _parse_int("٣") is ERR
    assert _cmp_double_int(9007199254740992.0, 9007199254740993) == 0 and _cmp_double_int(2.0 ** 63, I64_MAX) == 0
    assert _go_round(0.49999999999999994) == 0 and _go_round(-2.5) == -3 and math.copysign(1, _go_round(-0.4)) < 0
    assert math.copysign(1, _go_ceil(-0.5)) < 0 and math.copysign(1, _go_trunc(-0.5)) < 0 and _go_floor(-0.5) == -1
    assert _shr(-1, 1, True) == I64_MAX and _shl(1, 63, True) == I64_MIN and _shl(1, 64, True) == 0 and _shr(5, -1, True) is ERR
    assert [_fmt_g(x) for x in (1e21, 123456789.0, 100000.0, 1000000.0, 1e-5, 1e-4, 5e-324, -0.0, 0.1, 1e23, 2.5, 12.0)] == \
        ["1e+21", "1.23456789e+08", "100000", "1e+06", "1e-05", "0.0001", "5e-324", "-0", "0.1", "1e+23", "2.5", "12"]
    assert _fmt_fe(2.5, 0, "f") == "2" and _fmt_fe(0.125, 2, "f") == "0.12" and _fmt_fe(-0.0, 1, "f") == "-0.0" and _fmt_fe(INF, 3, "e") == "Infinity"
    assert _go_parse_duration("1h30m0.5s") == 5400500000000 and _go_parse_duration("-2562047h47m16.854775808s") == I64_MIN
    assert _go_parse_duration("2562047h47m16.854775808s") is ERR and _go_parse_duration("1.5") is ERR and _go_parse_duration("µs") is ERR
    assert _go_parse_duration("0.5μs") == 500 and _go_parse_duration(".5s") == 500000000
    a, b, c = _fma_sensitive(1, 9)[0]
    assert float(Fraction(a) * Fraction(b) + Fraction(c)) != a * b + c


@pytest.mark.parametrize("name", list(FAMILIES))
def test_family_vectors(name):
    """vector counts, outcome classes, ragged batches, and tables that take the unique-condition form with leaf programs"""
    probes = family(name)
    assert sum(len(p.vectors) for p in probes) >= MIN_VECTORS[name]
    assert set().union(*(p.outcomes() for p in probes)) == CLASSES[name]
    for p in probes:
        assert len(p.vectors) % 32 != 0
        assert all(repr(p.vectors[i][0]) != repr(p.vectors[i + 1][0]) for i in range(len(p.vectors) - 1))     # (repr: -0.0 is not 0.0)
        src, n_distinct = hostsim.generate_uc(p.ft.blob)
        assert "uc_atom_" in src and n_distinct == p.k, (p.conds, n_distinct)
        assert hostsim.generate(p.ft.blob) == ""      # not the block-shape form: the NVRTC unit holds the leaf programs


@pytest.mark.parametrize("name", list(FAMILIES))
def test_family_on_the_host_build(name, tmp_path):
    """every vector through the interpreter and the generated leaf programs, compiled for the host"""
    for j, p in enumerate(family(name)):
        b, want = p.batch, p.want()
        got = hostsim.check(p.ft.blob, b.columns, b.n, b.max_actions, NOW.ns, mode=1)
        _assert_same(p, got, want, "interpreter")
        d = tmp_path / str(j)
        d.mkdir()
        lib = hostsim.build_spec(p.ft.blob, str(d), uc=True)
        got = hostsim.check_spec(lib, p.ft.blob, b.columns, b.n, b.max_actions, NOW.ns, mode=4)
        _assert_same(p, got, want, "leaf programs")


@pytest.mark.parametrize("name", list(FAMILIES))
def test_family_against_oracle1(name):
    """oracle #1 on a seeded sample of about 2000 vectors per family"""
    probes = family(name)
    rng = random.Random(hash(name) & 0xFFFF)
    for p in probes:
        idx = sorted(rng.sample(range(len(p.vectors)), min(len(p.vectors), 2000 // len(probes))))
        o = CheckOracle(p.rt)
        names = {"EFFECT_ALLOW": 1, "EFFECT_DENY": 2, 1: 1, 2: 2}
        got = np.array([[names[o.check(p.request(i), NOW)["actions"][f"a{j}"]["effect"]] for j in range(p.k)] for i in idx], dtype=np.uint8)
        _assert_same(p, got, p.want(idx), "oracle #1", idx)


def _assert_same(p, got, want, what, idx=None):
    bad = np.argwhere(got[:, :want.shape[1]] != want)
    if len(bad):
        rows = []
        for r, c in bad[:6].tolist():
            i = idx[r] if idx is not None else r
            rows.append((p.conds[c // 2], p.vectors[i][0], p.vectors[i][1][c // 2], got[r, c // 2 * 2: c // 2 * 2 + 2].tolist()))
        pytest.fail(f"{p.family} / {what}: {len(bad)} effects differ from the exact reference, e.g. {rows}")


def test_narrow_columns_take_the_narrow_classes():
    p = family("narrow")[0]
    nb = NW.narrow_batch(p.batch, len(p.ft.manifest["slots"]))
    assert nb is not None
    slots = [tuple(s) for s in p.ft.manifest["slots"]]
    cls = np.asarray(nb.slot_class)
    assert cls[slots.index(("principal", "attr", "x"))] == NW.SLOT_F32
    assert cls[slots.index(("principal", "attr", "n"))] == NW.SLOT_U8_NUM


def test_nvrtc_unit_of_double_arithmetic_has_no_fused_multiply_add(tmp_path, monkeypatch):
    """a table whose conditions only multiply, add and subtract doubles: its NVRTC unit keeps DMUL + DADD (cel-go rounds each
    operation) and has no DFMA.  spec_compile writes the cubin to the cache directory; no device is needed."""
    from cerbos_b200 import capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    p = Probe("sass", [f"{expr} == P.attr.{name}" for name, expr, _ in FMA_OPS] + ["P.attr.a * P.attr.b == P.attr.m", "P.attr.a - P.attr.b == P.attr.d"],
              [({"a": 1.0, "b": 2.0, "c": 3.0, "n": -3.0, "r1": 5.0, "r2": 5.0, "r3": 5.0, "m": 2.0, "d": -1.0}, [HOLDS] * 5)])
    assert "uc_atom_" in hostsim.generate_uc(p.ft.blob)[0]
    monkeypatch.setenv("CERBOS_B200_CACHE_DIR", str(tmp_path))
    n, note = capi.compile_check(p.ft.blob)
    assert n > 0, note
    cubins = list(tmp_path.glob("spec_*.cubin"))
    assert len(cubins) == 1
    sass = subprocess.run([cuobjdump, "-sass", str(cubins[0])], capture_output=True, text=True, check=True).stdout
    ops = re.findall(r"\b(DMUL|DADD|DFMA)\b", sass)
    assert "DMUL" in ops and "DADD" in ops
    assert "DFMA" not in ops, [l for l in sass.split("\n") if "DFMA" in l][:5]


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def _context(monkeypatch, env):
    from cerbos_b200 import capi
    for k in ("CERBOS_B200_NO_JIT", "CERBOS_B200_UC"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return capi.Context(0)          # the switches are read when the context is made
    finally:
        for k in env:
            monkeypatch.delenv(k, raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FAMILIES))
def test_family_on_the_device(name, tmp_path, monkeypatch):
    """(a) the general kernel, (b) the NVRTC unique-condition kernel with leaf programs, (c) the metadata kernel on a
    4096-vector sample, (d) the narrow wire path for the printing and narrow-column families"""
    probes = family(name)
    monkeypatch.setenv("CERBOS_B200_CACHE_DIR", str(tmp_path))
    general = _context(monkeypatch, {"CERBOS_B200_NO_JIT": "1"})
    uc = _context(monkeypatch, {"CERBOS_B200_UC": "1"})
    try:
        tables = [(p, general.load_table(p.ft.blob), uc.load_table(p.ft.blob)) for p in probes]   # NVRTC compiles run side by side
        for p, tg, tu in tables:
            b, want = p.batch, p.want()
            got = tg.check(b.columns, b.n, b.max_actions, NOW.ns)
            cfg = general.last_kernel_config()
            assert not cfg["table_specialised"], cfg
            _assert_same(p, got, want, "general kernel")
            specialised, note = tu.wait_ready()
            assert specialised, note
            got = tu.check(b.columns, b.n, b.max_actions, NOW.ns)
            cfg = uc.last_kernel_config()
            assert cfg["table_specialised"] and cfg["unique_conditions"], cfg
            _assert_same(p, got, want, "unique-condition kernel")
            idx = sorted(random.Random(len(p.vectors)).sample(range(len(p.vectors)), min(len(p.vectors), 4096)))
            sb = Encoder(p.ft.manifest).encode([p.request(i) for i in idx])
            eff, _, _ = tu.check_meta(sb.columns, sb.n, sb.max_actions, NOW.ns)
            _assert_same(p, eff, p.want(idx), "metadata kernel", idx)
            if name in ("printing", "narrow"):
                nb = NW.narrow_batch(b, len(p.ft.manifest["slots"]))
                assert nb is not None
                got = tu.check_narrow(nb, NOW.ns)
                _assert_same(p, got, want, "narrow path")
        for _, tg, tu in tables:
            tg.release()
            tu.release()
    finally:
        general.close()
        uc.close()
