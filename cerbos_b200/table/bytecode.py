"""CEL condition trees -> device bytecode (host side, at table build).

Replaces, for the GPU path, what the reference does at evaluation time with
cel-go's tree-walking interpreter: ``SatisfiesCondition`` /
``evaluateBoolCELExpr`` (internal/ruletable/ruletable.go:1346-1441, 1467-1486)
over the environment of internal/conditions/cel.go:62-75.

What is lowered
  * condition trees all/any/none/expr with the reference's leaf rule
    "error or non-bool => false" (TO_COND);
  * request paths (``P.attr.x``, ``R.attr.a.b``, ``request.aux_data.jwt.aud`` ...)
    -> attribute *slots*: the batch encoder extracts the value per request into a
    NaN-boxed 8-byte column (SURVEY.md 8(d));
  * ``C.x`` / ``constants.x`` / ``G.x`` / ``globals.x`` folded to literals; ``V.x`` /
    ``variables.x`` inlined (policy variables are pure; an erroring variable is
    "unset" in the reference, ruletable.go:1325-1332, and an inlined erroring
    expression is equally an error; ``has(V.x)`` -> NOERR);
  * operators, ``in``, index/select, size, startsWith/endsWith/contains,
    hasIntersection/isSubset, all/exists/exists_one (1- and 2-variable),
    ternary, numeric/timestamp/duration conversions, now()/timeSince(), format() with a constant format string and
    strings.quote (ext.Strings).

Anything else raises :class:`Unsupported` -- table build fails loudly; there is no
silent per-request divergence and no CPU fallback (SURVEY.md 8(b)).
"""
from __future__ import annotations

import math
import struct

from ..cel.ast import Call, Const, Ident, ListLit, Macro, MapLit, Node, Select, UInt
from ..policy.model import Cond, Params
from . import layout as L
from .consts import parse_cidr, parse_duration_ns, parse_timestamp_ns

OP = L.OPS
T = L.TAGS


class Unsupported(Exception):
    """The expression cannot be lowered exactly to device bytecode."""


_PRINCIPAL_FIELDS = {"id", "roles", "attr", "policy_version", "scope"}
_RESOURCE_FIELDS = {"kind", "id", "attr", "policy_version", "scope"}
_ALIASES = {"policyVersion": "policy_version", "auxData": "aux_data",
            "effectiveDerivedRoles": "effective_derived_roles"}


def f64_bits(d: float) -> int:
    if math.isnan(d):
        return L.V64_CANON_NAN
    return struct.unpack("<Q", struct.pack("<d", d))[0]


def box(tag: int, payload: int = 0) -> int:
    return ((L.V64_BOX_BASE | tag) << 48) | (payload & ((1 << 48) - 1))


class StringTable:
    def __init__(self):
        self.ids = {}
        self.items = []

    def intern(self, s: str) -> int:
        i = self.ids.get(s)
        if i is None:
            i = len(self.items)
            self.ids[s] = i
            self.items.append(s)
        return i

    def __len__(self):
        return len(self.items)


class ConstVal:
    """Compile-time constant: (tag, bits) plus the Python value for further folding."""
    __slots__ = ("tag", "bits", "py")

    def __init__(self, tag, bits, py=None):
        self.tag = tag
        self.bits = bits & 0xFFFFFFFFFFFFFFFF
        self.py = py


class TableBuilderCtx:
    """Pools shared by every program of one table."""

    def __init__(self, globals_=None):
        self.strings = StringTable()
        self.consts: list[ConstVal] = []
        self._const_ix = {}
        self.theap: list[int] = []
        self._heap_ix = {}
        self.slots: dict[tuple, int] = {}
        self.globals = globals_ or {}
        self.uses_pid = False
        self.uses_now = False
        self.max_stack = 0
        self.max_loop_depth = 0
        self.n_vars = 0
        self.uses_runtime = False

    # -- pools
    def slot(self, path: tuple) -> int:
        i = self.slots.get(path)
        if i is None:
            i = len(self.slots)
            self.slots[path] = i
        return i

    def const_index(self, cv: ConstVal) -> int:
        k = (cv.tag, cv.bits)
        i = self._const_ix.get(k)
        if i is None:
            i = len(self.consts)
            self._const_ix[k] = i
            self.consts.append(cv)
        return i

    def v64_of(self, v, native_ints: bool) -> int:
        """Python constant -> NaN-boxed heap element."""
        if v is None:
            return box(L.V64_NULL)
        if isinstance(v, bool):
            return box(L.V64_BOOL, int(v))
        if isinstance(v, UInt):
            raise Unsupported("uint element in constant list/map")
        if isinstance(v, int):
            if not native_ints:
                return f64_bits(float(v))
            if not (-(1 << 47) <= v < (1 << 47)):
                raise Unsupported("int constant too large for list element")
            return box(L.V64_INT, v)
        if isinstance(v, float):
            return f64_bits(v)
        if isinstance(v, str):
            return box(L.V64_STRING, self.strings.intern(v))
        if isinstance(v, (list, tuple)):
            return box(L.V64_LIST, self.heap_list([self.v64_of(x, native_ints) for x in v]))
        if isinstance(v, dict):
            return box(L.V64_MAP, self.heap_map(v, native_ints))
        raise Unsupported(f"constant of type {type(v).__name__}")

    def _heap_put(self, words: list) -> int:
        k = tuple(words)
        off = self._heap_ix.get(k)
        if off is None:
            off = len(self.theap)
            self._heap_ix[k] = off
            self.theap.extend(words)
        return off

    def heap_list(self, elems_v64: list) -> int:
        return self._heap_put([len(elems_v64)] + list(elems_v64))

    def heap_map(self, d: dict, native_ints: bool) -> int:
        keys, vals = [], []
        for k, v in d.items():
            if isinstance(k, str):
                keys.append(box(L.V64_STRING, self.strings.intern(k)))
            elif isinstance(k, (bool, int, float)) and not isinstance(k, UInt) and native_ints:
                keys.append(self.v64_of(k, True))       # CEL map literal with bool / int / double keys
            else:
                raise Unsupported("map key that is not a string, int, double or bool")
            vals.append(self.v64_of(v, native_ints))
        return self._heap_put([len(keys)] + keys + vals)

    def const_from_py(self, v, native_ints: bool) -> ConstVal:
        """JSON-ish Python value -> ConstVal. native_ints=False: numbers are doubles
        (google.protobuf.Value); True: Python ints are CEL ints (CEL literals, Go-native globals)."""
        if v is None:
            return ConstVal(T["NULL"], 0, None)
        if isinstance(v, bool):
            return ConstVal(T["BOOL"], int(v), v)
        if isinstance(v, UInt):
            return ConstVal(T["UINT"], int(v), v)
        if isinstance(v, int):
            if native_ints:
                return ConstVal(T["INT"], v, v)
            return ConstVal(T["DOUBLE"], f64_bits(float(v)), float(v))
        if isinstance(v, float):
            return ConstVal(T["DOUBLE"], f64_bits(v), v)
        if isinstance(v, str):
            return ConstVal(T["STRING"], self.strings.intern(v), v)
        if isinstance(v, bytes):
            raise Unsupported("bytes constants")
        if isinstance(v, (list, tuple)):
            return ConstVal(T["LIST"], self.heap_list([self.v64_of(x, native_ints) for x in v]), list(v))
        if isinstance(v, dict):
            return ConstVal(T["MAP"], self.heap_map(v, native_ints), dict(v))
        raise Unsupported(f"constant of type {type(v).__name__}")


_ZONE_CACHE: dict = {}


def iana_zone_words(name: str):
    """Transition table of an IANA zone for the device: [n, first covered second, last covered second, then n pairs
    (UTC second from which the offset applies, offset east of UTC in seconds as two's complement)].  Built from the host's
    tz database (zoneinfo; Go's time.LoadLocation reads the same data); None for an unknown zone.  Instants outside
    1900-01-01 .. 2100-01-01 are not covered (the device then fails the call loudly)."""
    if name in _ZONE_CACHE:
        return _ZONE_CACHE[name]
    import datetime as _dt
    import zoneinfo
    zi = None
    cand = name
    for _ in range(3):
        try:
            zi = zoneinfo.ZoneInfo(cand)
            break
        except Exception:  # noqa: BLE001 -- backward-compatible link names live in tzdata.zi on some hosts
            link = None
            try:
                with open("/usr/share/zoneinfo/tzdata.zi", encoding="utf-8") as f:
                    for ln in f:
                        parts = ln.split()
                        if len(parts) == 3 and parts[0] == "L" and parts[2] == cand:
                            link = parts[1]
                            break
            except OSError:
                pass
            if link is None:
                break
            cand = link
    if zi is None:
        _ZONE_CACHE[name] = None
        return None
    utc = _dt.timezone.utc

    def off(sec):
        return int(_dt.datetime.fromtimestamp(sec, tz=utc).astimezone(zi).utcoffset().total_seconds())

    lo = int(_dt.datetime(1900, 1, 1, tzinfo=utc).timestamp())
    hi = int(_dt.datetime(2100, 1, 1, tzinfo=utc).timestamp())
    pairs = [(lo, off(lo))]
    t, cur = lo, pairs[0][1]
    step = 86400
    while t < hi:
        nt = min(t + step, hi)
        o = off(nt)
        if o != cur:
            a, b = t, nt          # offset(a) == cur, offset(b) != cur: bisect to the first second of the new offset
            while b - a > 1:
                m = (a + b) // 2
                if off(m) == cur:
                    a = m
                else:
                    b = m
            cur = off(b)
            pairs.append((b, cur))
            t = b
            continue
        t = nt
    words = [len(pairs), lo & 0xFFFFFFFFFFFFFFFF, hi & 0xFFFFFFFFFFFFFFFF]
    for sec, o in pairs:
        words += [sec & 0xFFFFFFFFFFFFFFFF, o & 0xFFFFFFFFFFFFFFFF]
    _ZONE_CACHE[name] = words
    return words


class _Static:
    """Result of static path analysis."""
    __slots__ = ("kind", "path", "value", "native")

    def __init__(self, kind, path=None, value=None, native=False):
        self.kind = kind      # 'slot' | 'const' | 'missing' | 'pid'
        self.path = path
        self.value = value
        self.native = native


_MISSING = object()


class ProgramCompiler:
    def __init__(self, ctx: TableBuilderCtx, params: Params | None):
        self.ctx = ctx
        self.constants = (params.constants if params else {}) or {}
        self.var_defs = {v.name: v.expr for v in (params.variables if params else [])}
        self.code: list[list] = []
        self.sp = 0
        self.loop_vars: list[dict] = []   # stack of {name: var index}
        self.inlining: list[str] = []
        self.stack_limit = L.MAX_STACK    # value programs (rule outputs) run with the deeper OUT_MAX_STACK

    # ---------------------------------------------------------------- emit helpers
    def emit(self, op, a=0, b=0, c=0, delta=0):
        self.code.append([OP[op], a, b, c])
        self.sp += delta
        if self.sp > self.ctx.max_stack and self.stack_limit == L.MAX_STACK:
            self.ctx.max_stack = self.sp
        if self.sp > self.stack_limit:
            raise Unsupported("expression needs a deeper evaluation stack than the device provides")
        return len(self.code) - 1

    def here(self):
        return len(self.code)

    def patch(self, at, field, val):
        self.code[at][{"a": 1, "b": 2, "c": 3}[field]] = val

    def push_const(self, cv: ConstVal):
        self.emit("CONST", c=self.ctx.const_index(cv), delta=1)

    # ---------------------------------------------------------------- conditions
    def compile_cond(self, cond: Cond):
        """Leaves a plain BOOL on the stack."""
        if cond.op == "expr":
            self.expr(cond.expr.ast)
            self.emit("TO_COND")
            return
        kids = cond.children
        if not kids:
            # all[] -> true ; any[] -> false ; none[] -> true
            self.push_const(ConstVal(T["BOOL"], 0 if cond.op == "any" else 1))
            return
        jumps = []
        for i, ch in enumerate(kids):
            self.compile_cond(ch)
            if i > 0:
                self.emit("AND" if cond.op == "all" else "OR", delta=-1)
            if i < len(kids) - 1:
                jumps.append(self.emit("JF_KEEP" if cond.op == "all" else "JT_KEEP"))
        end = self.here()
        for j in jumps:
            self.patch(j, "c", end)
        if cond.op == "none":
            self.emit("COND_NOT")

    # ---------------------------------------------------------------- static paths
    def _lookup_var(self, name):
        for frame in reversed(self.loop_vars):
            if name in frame:
                return frame[name]
        return None

    def _static(self, n: Node):
        """Tries to resolve `n` without emitting code. Returns _Static or None."""
        segs = []
        cur = n
        while True:
            if isinstance(cur, Select) and not cur.test_only:
                segs.append(cur.field)
                cur = cur.operand
            elif (isinstance(cur, Call) and cur.fn == "_[_]" and isinstance(cur.args[1], Const)
                  and isinstance(cur.args[1].value, str)):
                segs.append(cur.args[1].value)
                cur = cur.args[0]
            else:
                break
        if not isinstance(cur, Ident) or self._lookup_var(cur.name) is not None:
            return None
        segs.reverse()
        root = cur.name
        if root in ("request", "R", "P"):
            if root == "R":
                segs = ["resource"] + segs
            elif root == "P":
                segs = ["principal"] + segs
            return self._request_path(segs)
        if root in ("C", "constants"):
            return self._const_path(self.constants, segs, native=False, what="constants")
        if root in ("G", "globals"):
            return self._const_path(self.ctx.globals, segs, native=True, what="globals")
        return None

    def _request_path(self, segs):
        if not segs:
            raise Unsupported("bare `request` value")
        first = _ALIASES.get(segs[0], segs[0])
        if first in ("principal", "resource"):
            if len(segs) < 2:
                raise Unsupported(f"bare `request.{first}` message value")
            fld = _ALIASES.get(segs[1], segs[1])
            allowed = _PRINCIPAL_FIELDS if first == "principal" else _RESOURCE_FIELDS
            if fld not in allowed:
                raise Unsupported(f"unknown field request.{first}.{segs[1]}")
            path = (first, fld) + tuple(segs[2:])
            if fld != "attr" and len(segs) > 2:
                if fld == "roles":
                    raise Unsupported("field selection on request.principal.roles")
                raise Unsupported(f"field selection on string request.{first}.{fld}")
            if path == ("principal", "id"):
                return _Static("pid")
            return _Static("slot", path=path)
        if first == "aux_data":
            if len(segs) < 2:
                raise Unsupported("bare `request.aux_data` message value")
            if segs[1] != "jwt":
                raise Unsupported(f"unknown field request.aux_data.{segs[1]}")
            return _Static("slot", path=("aux_data", "jwt") + tuple(segs[2:]))
        raise Unsupported(f"unknown field request.{segs[0]}")

    def _const_path(self, root, segs, native, what):
        if not segs:
            return _Static("const", value=dict(root), native=native)
        cur = root
        for s in segs:
            if isinstance(cur, dict) and s in cur:
                cur = cur[s]
            else:
                return _Static("missing")  # no such key -> CEL error at run time
        return _Static("const", value=cur, native=native)

    def _push_static(self, st: _Static):
        if st.kind == "slot":
            self.emit("SLOT", c=self.ctx.slot(st.path), delta=1)
        elif st.kind == "pid":
            self.ctx.uses_pid = True
            self.emit("PID", delta=1)
        elif st.kind == "const":
            self.push_const(self.ctx.const_from_py(st.value, st.native))
        else:
            self.push_const(ConstVal(T["ERR"], 0))

    # ---------------------------------------------------------------- expressions
    def expr(self, n: Node):
        if isinstance(n, Const):
            v = n.value
            if isinstance(v, bytes):
                try:        # the string table holds UTF-8 text: a bytes literal that is valid UTF-8 is that string, retagged
                    text = v.decode("utf-8")
                except UnicodeDecodeError:
                    raise Unsupported("bytes literal that is not valid UTF-8") from None
                self.push_const(self.ctx.const_from_py(text, native_ints=True))
                self.emit("FN", a=L.FNS["TO_BYTES"], b=1)
                return
            self.push_const(self.ctx.const_from_py(v, native_ints=True))
            return
        if isinstance(n, Ident):
            vi = self._lookup_var(n.name)
            if vi is not None:
                self.emit("VAR", a=vi, delta=1)
                return
            if n.name in ("runtime",):
                raise Unsupported("`runtime` (effectiveDerivedRoles) in conditions")
            if n.name in L.TYPE_CODES:        # a type name as a value: `type(x) == string`
                self.push_const(ConstVal(T["TYPE"], L.TYPE_CODES[n.name]))
                return
            st = self._static(n)
            if st is not None:
                self._push_static(st)
                return
            raise Unsupported(f"identifier `{n.name}` as a value")
        if isinstance(n, Select):
            return self._select(n)
        if isinstance(n, Call):
            return self._call(n)
        if isinstance(n, (ListLit, MapLit)):
            try:
                value = self._literal_value(n)
            except Unsupported:
                return self._dynamic_literal(n)
            self.push_const(self.ctx.const_from_py(value, native_ints=True))
            return
        if isinstance(n, Macro):
            return self._macro(n)
        raise Unsupported(f"node {type(n).__name__}")

    def _dynamic_literal(self, n: Node):
        """[e0, e1 ...] / {k0: v0 ...} with elements computed at run time: built in the device's scratch arena."""
        if isinstance(n, ListLit):
            if len(n.elems) > 12:
                raise Unsupported("list literal with more than 12 run-time elements")
            for e in n.elems:
                self.expr(e)
            self.emit("MKLIST", c=len(n.elems), delta=1 - len(n.elems))
            return
        if len(n.entries) > 6:
            raise Unsupported("map literal with more than 6 run-time entries")
        for k, v in n.entries:
            self.expr(k)
            self.expr(v)
        self.emit("MKMAP", c=len(n.entries), delta=1 - 2 * len(n.entries))

    def _literal_value(self, n: Node):
        if isinstance(n, Const):
            if isinstance(n.value, bytes):
                raise Unsupported("bytes literal")
            return n.value
        if isinstance(n, ListLit):
            return [self._literal_value(e) for e in n.elems]
        if isinstance(n, MapLit):
            out = {}
            for k, v in n.entries:
                kv = self._literal_value(k)
                if not isinstance(kv, (str, bool, int, float)) or isinstance(kv, UInt):
                    raise Unsupported("map literal key that is not a string, int, double or bool")
                if kv in out:
                    raise Unsupported("repeated key in map literal")
                out[kv] = self._literal_value(v)
            return out
        st = self._static(n) if isinstance(n, (Select, Ident, Call)) else None
        if st is not None and st.kind == "const" and st.native:
            return st.value
        raise Unsupported("list / map literal with non-constant elements")


    def _var_inline(self, name: str):
        if name not in self.var_defs:
            # undefined variables are a policy compile error in the reference (compile/variables.go)
            raise Unsupported(f"undefined variable '{name}'")
        if name in self.inlining:
            raise Unsupported(f"cyclic variable '{name}'")
        self.inlining.append(name)
        saved, self.loop_vars = self.loop_vars, []   # variable bodies do not see comprehension variables
        self.expr(self.var_defs[name].ast)
        self.loop_vars = saved
        self.inlining.pop()

    def _is_var_ref(self, n: Node):
        return (isinstance(n, Select) and not n.test_only and isinstance(n.operand, Ident)
                and n.operand.name in ("V", "variables") and self._lookup_var(n.operand.name) is None)

    def _select(self, n: Select):
        if n.test_only:
            return self._has(n)
        if self._is_var_ref(n):
            return self._var_inline(n.field)
        st = self._static(n)
        if st is not None:
            return self._push_static(st)
        if isinstance(n.operand, Ident) and n.operand.name == "runtime" and self._lookup_var("runtime") is None:
            if n.field not in ("effectiveDerivedRoles", "effective_derived_roles"):
                raise Unsupported(f"unknown field runtime.{n.field}")
            self.ctx.uses_runtime = True
            self.emit("RUNTIME_EDR", delta=1)
            return
        self.expr(n.operand)
        self.emit("SELECT", c=self.ctx.strings.intern(n.field))

    def _has(self, n: Select):
        op = n.operand
        if isinstance(op, Ident) and op.name in ("V", "variables") and self._lookup_var(op.name) is None:
            if n.field not in self.var_defs:
                self.push_const(ConstVal(T["BOOL"], 0))
                return
            self._var_inline(n.field)
            self.emit("NOERR")
            return
        full = Select(op, n.field)
        st = self._static(full)
        if st is not None:
            if st.kind == "slot":
                if len(st.path) <= 2:
                    raise Unsupported("has() on a request message field")
                self.emit("HAS_SLOT", c=self.ctx.slot(st.path), delta=1)
                return
            if st.kind == "pid":
                raise Unsupported("has() on a request message field")
            if st.kind == "const":
                self.push_const(ConstVal(T["BOOL"], 1))
                return
            # missing: has() is false only if the parent exists
            pst = self._static(op)
            if pst is not None and pst.kind == "const" and isinstance(pst.value, dict):
                self.push_const(ConstVal(T["BOOL"], 0))
            else:
                self.push_const(ConstVal(T["ERR"], 0))
            return
        self.expr(op)
        self.emit("HAS", c=self.ctx.strings.intern(n.field))

    _BIN = {"_==_": "EQ", "_!=_": "NE", "_<_": "LT", "_<=_": "LE", "_>_": "GT", "_>=_": "GE",
            "_+_": "ADD", "_-_": "SUB", "_*_": "MUL", "_/_": "DIV", "_%_": "MOD", "@in": "IN", "_[_]": "INDEX"}
    _STR2 = {"startsWith": "STARTS_WITH", "endsWith": "ENDS_WITH", "contains": "CONTAINS"}
    _LIST2 = {"hasIntersection": "HAS_INTERSECTION", "has_intersection": "HAS_INTERSECTION",
              "isSubset": "IS_SUBSET", "is_subset": "IS_SUBSET"}
    _CONV = {"int": "INT", "uint": "UINT", "double": "DOUBLE", "timestamp": "TIMESTAMP", "duration": "DURATION",
             "dyn": "DYN", "id": "DYN"}

    def _simple(self, n: Node):
        """('slot', path) | ('const', ConstVal) | ('pid',) for operands a super-instruction can
        address; no pool side effects (allocation happens when the fused op is emitted)."""
        if isinstance(n, Const) and not isinstance(n.value, bytes):
            return ("const", (n.value, True))
        if isinstance(n, ListLit):
            try:
                return ("const", (self._literal_value(n), True))
            except Unsupported:
                return None
        if isinstance(n, (Select, Ident, Call)) and not (isinstance(n, Select) and n.test_only):
            if isinstance(n, Call) and n.fn != "_[_]":
                return None
            if self._is_var_ref(n):
                d = self.var_defs.get(n.field)
                if d is not None and isinstance(d.ast, Const) and not isinstance(d.ast.value, bytes):
                    return ("const", (d.ast.value, True))
                return None
            try:
                st = self._static(n)
            except Unsupported:
                return None
            if st is None:
                return None
            if st.kind == "slot":
                return ("slot", st.path)
            if st.kind == "pid":
                return ("pid",)
            if st.kind == "const":
                return ("const", (st.value, st.native))
        return None

    def _slot_ix(self, path):
        s = self.ctx.slot(path)
        if s > 0xFFFF:
            raise Unsupported("too many attribute slots")
        return s

    def _const_ix(self, desc):
        return self.ctx.const_index(self.ctx.const_from_py(desc[0], desc[1]))

    def _try_fused(self, fn, a, b) -> bool:
        if fn not in L.CMP_INDEX and fn != "@in":
            return False
        sa, sb = self._simple(a), self._simple(b)
        if sa is None or sb is None:
            return False
        ka, kb = sa[0], sb[0]
        if fn in L.CMP_INDEX:
            ci = L.CMP_INDEX[fn]
            swap = {0: 0, 1: 1, 2: 4, 3: 5, 4: 2, 5: 3}
            if ka == "slot" and kb == "const":
                self.emit("CMP_SLOT_CONST", a=ci, b=self._slot_ix(sa[1]), c=self._const_ix(sb[1]), delta=1)
            elif ka == "const" and kb == "slot":
                self.emit("CMP_SLOT_CONST", a=swap[ci], b=self._slot_ix(sb[1]), c=self._const_ix(sa[1]), delta=1)
            elif ka == "slot" and kb == "slot":
                self.emit("CMP_SLOT_SLOT", a=ci, b=self._slot_ix(sa[1]), c=self._slot_ix(sb[1]), delta=1)
            elif ka == "slot" and kb == "pid":
                self.ctx.uses_pid = True
                self.emit("CMP_SLOT_PID", a=ci, b=self._slot_ix(sa[1]), delta=1)
            elif ka == "pid" and kb == "slot":
                self.ctx.uses_pid = True
                self.emit("CMP_SLOT_PID", a=swap[ci], b=self._slot_ix(sb[1]), delta=1)
            else:
                return False
            return True
        if ka == "slot" and kb == "const":
            self.emit("IN_SLOT_CONST", b=self._slot_ix(sa[1]), c=self._const_ix(sb[1]), delta=1)
            return True
        if ka == "const" and kb == "slot":
            self.emit("IN_CONST_SLOT", b=self._slot_ix(sb[1]), c=self._const_ix(sa[1]), delta=1)
            return True
        return False

    def _call(self, n: Call):
        fn = n.fn
        args = ([n.target] if n.target is not None else []) + n.args
        if fn == "_&&_" or fn == "_||_":
            self.expr(args[0])
            j = self.emit("JF_KEEP" if fn == "_&&_" else "JT_KEEP")
            self.expr(args[1])
            self.emit("AND" if fn == "_&&_" else "OR", delta=-1)
            self.patch(j, "c", self.here())
            return
        if fn == "_?_:_":
            self.expr(args[0])
            t = self.emit("TERN", delta=-1)
            sp0 = self.sp
            self.expr(args[1])
            j = self.emit("JMP")
            self.patch(t, "c", self.here())
            self.sp = sp0
            self.expr(args[2])
            end = self.here()
            if end > 0xFFFF:
                raise Unsupported("program too long")
            self.patch(t, "b", end)
            self.patch(j, "c", end)
            return
        if fn == "@hier_join" and len(args) == 1:
            self.expr(args[0])
            self.emit("FN", a=L.FNS["HIER_JOIN"], b=1)
            return
        if fn == "_[_]" and len(args) == 2:
            h = self._hier(args[0])
            if h:       # hierarchy(..)[i]: the i-th part
                self.expr(h[0])
                self.expr(args[1])
                self.emit("CONST", c=self.ctx.const_index(ConstVal(T["STRING"], h[1])), delta=1)
                self.emit("FN", a=L.FNS["HIER_AT"], b=3, delta=-2)
                return
        if self._hier_call(fn, args):
            return
        if fn == "@in" and len(args) == 2 and isinstance(args[1], Call) and args[1].fn == "split" and args[1].target is not None \
                and len(args[1].args) == 1 and isinstance(args[1].args[0], Const) and isinstance(args[1].args[0].value, str) \
                and args[1].args[0].value:
            # x in s.split("sep"): membership among the separated tokens, fused (the list is never built)
            did = self.ctx.strings.intern(args[1].args[0].value)
            if did > 0xFFFF:
                raise Unsupported("too many table strings for a split separator")
            self.expr(args[0])
            self.expr(args[1].target)
            self.emit("IN_SPLIT", b=did, delta=-1)
            return
        if fn == "_[_]" or fn in L.CMP_INDEX or fn == "@in":
            st = self._static(n) if fn == "_[_]" else None
            if st is not None:
                return self._push_static(st)
            if len(args) == 2 and self._try_fused(fn, args[0], args[1]):
                return
        if fn in self._BIN and len(args) == 2:
            self.expr(args[0])
            self.expr(args[1])
            self.emit(self._BIN[fn], delta=-1)
            return
        if fn == "!_" and len(args) == 1:
            self.expr(args[0])
            self.emit("NOT")
            return
        if fn == "-_" and len(args) == 1:
            self.expr(args[0])
            self.emit("NEG")
            return
        if fn == "size" and len(args) == 1:
            self.expr(args[0])
            self.emit("SIZE")
            return
        if fn in self._STR2 and len(args) == 2:
            self.expr(args[0])
            self.expr(args[1])
            self.emit(self._STR2[fn], delta=-1)
            return
        if fn in self._LIST2 and len(args) == 2:
            self.expr(args[0])
            self.expr(args[1])
            self.emit(self._LIST2[fn], delta=-1)
            return
        if fn in ("timestamp", "duration") and len(args) == 1 and isinstance(args[0], Const) \
                and isinstance(args[0].value, str):
            try:
                if fn == "timestamp":
                    self.push_const(ConstVal(T["TS"], parse_timestamp_ns(args[0].value)))
                else:
                    self.push_const(ConstVal(T["DUR"], parse_duration_ns(args[0].value)))
            except ValueError:
                self.push_const(ConstVal(T["ERR"], 0))
            return
        if fn in self._CONV and len(args) == 1:
            self.expr(args[0])
            self.emit(self._CONV[fn])
            return
        if fn == "inIPAddrRange" and len(args) == 2:
            if not (isinstance(args[1], Const) and isinstance(args[1].value, str)):
                raise Unsupported("inIPAddrRange with a non-constant CIDR")
            cidr = parse_cidr(args[1].value)
            if cidr is None:
                # invalid CIDR text is a CEL error whatever the address is (cerbos_lib.go:472-484)
                self.push_const(ConstVal(T["ERR"], 0))
                return
            self.expr(args[0])
            self.emit("IN_IP_RANGE", c=self.ctx._heap_put(list(cidr)))
            return
        if fn in L.TS_FIELDS and len(args) in (1, 2):
            off, tzform = 0, 0
            if len(args) == 2:
                # a constant fixed offset ("-05:00", "UTC"); IANA zone names would need a tz database on the device
                tz = args[1]
                if not (isinstance(tz, Const) and isinstance(tz.value, str)):
                    raise Unsupported("timestamp accessor with a non-constant time zone")
                tzs = tz.value
                if ":" in tzs:
                    ind = tzs.index(":")
                    try:
                        hr, mn = int(tzs[:ind]), int(tzs[ind + 1:])
                    except ValueError:
                        self.expr(args[0])          # invalid zone text: a CEL error whatever the timestamp is
                        self.emit("TS_GET", a=0xFF)
                        return
                    off = (hr * 60 - mn if tzs[0] == "-" else hr * 60 + mn) * 60
                elif tzs not in ("UTC", ""):
                    # an IANA zone name: its UTC-offset transitions 1900..2100 go into the table (built from the host's tz database)
                    words = iana_zone_words(tzs)
                    if words is None:
                        self.expr(args[0])          # unknown zone: a CEL error whatever the timestamp is
                        self.emit("TS_GET", a=0xFF)
                        return
                    self.expr(args[0])
                    self.emit("TS_GET", a=L.TS_FIELDS[fn], b=2, c=self.ctx._heap_put(words))
                    return
                tzform = 1
                if not -(1 << 31) <= off < (1 << 31):
                    raise Unsupported("time zone offset out of range")
            self.expr(args[0])
            self.emit("TS_GET", a=L.TS_FIELDS[fn], b=tzform, c=off & 0xFFFFFFFF)
            return
        if fn == "now" and not args:
            self.ctx.uses_now = True
            self.emit("NOW", delta=1)
            return
        if fn == "timeSince" and len(args) == 1:
            self.ctx.uses_now = True
            self.emit("NOW", delta=1)
            self.expr(args[0])
            self.emit("SUB", delta=-1)
            return
        if fn == "matches" and len(args) == 2:
            # RE2 search: a constant pattern becomes a byte-level DFA table at table build (cel/regex_dfa.py)
            from ..cel.regex_dfa import RegexError, RegexUnsupported, compile_dfa, dfa_words
            if not (isinstance(args[1], Const) and isinstance(args[1].value, str)):
                raise Unsupported("matches() with a non-constant pattern")
            try:
                words = dfa_words(compile_dfa(args[1].value))
            except RegexUnsupported as e:
                raise Unsupported(f"regular expression: {e}") from e
            except RegexError:
                self.push_const(ConstVal(T["ERR"], 0))    # an invalid pattern is an error whatever the text is
                return
            self.expr(args[0])
            self.emit("MATCHES", c=self.ctx._heap_put(words))
            return
        if self._spiffe_call(n, fn, args):
            return
        if fn in self._MATH and (len(args) in self._MATH[fn][1] or (self._MATH[fn][1] == () and 1 <= len(args) <= 16)):
            # cel-go ext.Math: scalar functions; greatest / least take one number, one list or several numbers.  The macro
            # behind greatest / least refuses literal arguments that are not numbers at compile time (ext/math.go)
            if self._MATH[fn][1] == ():
                for a in args:
                    bad_literal = isinstance(a, (MapLit, Macro)) or (isinstance(a, ListLit) and len(args) > 1) or \
                        (isinstance(a, Const) and (isinstance(a.value, (str, bytes, bool)) or a.value is None))
                    if bad_literal:
                        raise Unsupported(f"{fn}: a literal argument that is not a number (compile error in the reference)")
            for a in args:
                self.expr(a)
            self.emit("FN", a=L.FNS[self._MATH[fn][0]], b=len(args), delta=1 - len(args))
            return
        if fn == "format" and n.target is not None and len(n.args) == 1:
            return self._format(n.target, n.args[0])
        if fn in self._FN and len(args) in self._FN[fn][1]:
            # string / list producing functions (ext.Strings, ext.Lists, Cerbos except / intersect): results live in the
            # device's per-thread scratch arena
            for a in args:
                self.expr(a)
            self.emit("FN", a=L.FNS[self._FN[fn][0]], b=len(args), delta=1 - len(args))
            return
        raise Unsupported(f"function `{fn}` with {len(args)} argument(s)")

    _MATH = {"math.greatest": ("MATH_GREATEST", ()), "math.least": ("MATH_LEAST", ()), "math.ceil": ("MATH_CEIL", (1,)),
             "math.floor": ("MATH_FLOOR", (1,)), "math.round": ("MATH_ROUND", (1,)), "math.trunc": ("MATH_TRUNC", (1,)),
             "math.abs": ("MATH_ABS", (1,)), "math.sign": ("MATH_SIGN", (1,)), "math.isNaN": ("MATH_ISNAN", (1,)),
             "math.isInf": ("MATH_ISINF", (1,)), "math.isFinite": ("MATH_ISFINITE", (1,)), "math.bitAnd": ("MATH_BITAND", (2,)),
             "math.bitOr": ("MATH_BITOR", (2,)), "math.bitXor": ("MATH_BITXOR", (2,)), "math.bitNot": ("MATH_BITNOT", (1,)),
             "math.bitShiftLeft": ("MATH_SHL", (2,)), "math.bitShiftRight": ("MATH_SHR", (2,)), "math.sqrt": ("MATH_SQRT", (1,))}
    _FN = {"bytes": ("TO_BYTES", (1,)), "string": ("TO_STRING", (1,)), "bool": ("TO_BOOL", (1,)), "type": ("TYPE_OF", (1,)), "base64.encode": ("B64ENC", (1,)), "base64.decode": ("B64DEC", (1,)),
           "lowerAscii": ("LOWER", (1,)), "upperAscii": ("UPPER", (1,)), "trim": ("TRIM", (1,)), "charAt": ("CHARAT", (2,)),
           "indexOf": ("INDEXOF", (2, 3)), "lastIndexOf": ("LASTINDEXOF", (2, 3)), "substring": ("SUBSTRING", (2, 3)),
           "replace": ("REPLACE", (3, 4)), "split": ("SPLIT", (2, 3)), "join": ("JOIN", (1, 2)), "reverse": ("REVERSE", (1,)),
           "except": ("EXCEPT", (2,)), "intersect": ("INTERSECT", (2,)), "sort": ("SORT", (1,)), "slice": ("SLICE", (3,)),
           "flatten": ("FLATTEN", (1, 2)), "distinct": ("DISTINCT", (1,)), "lists.range": ("RANGE", (1,)),
           "strings.quote": ("QUOTE", (1,))}

    def _format(self, target: Node, arg: Node):
        """fmt.format(args) (ext.Strings) with a constant fmt: its clauses are parsed here, once, into a THEAP record (layout
        FORMAT).  A list-literal `args` of up to FORMAT_MAX_STACK_ARGS elements is compiled element by element onto the stack,
        so no list is built at run time and the condition stays within the leaf-program translator; a longer literal (or any
        other list value) is one operand, the list."""
        fmt = None
        if isinstance(target, Const) and isinstance(target.value, str):
            fmt = target.value
        else:
            s = self._simple(target)
            if s is not None and s[0] == "const" and isinstance(s[1][0], str):
                fmt = s[1][0]
        if fmt is None:
            raise Unsupported("format() with a format string that is not a constant")
        items = parse_format(fmt)
        if items is None:
            # a clause that cannot be parsed is an error whatever the arguments are (every clause is reached)
            self.push_const(ConstVal(T["ERR"], 0))
            return
        words = [len(items)]
        for it in items:
            if it[0] == "lit":
                words.append(self.ctx.strings.intern(it[1]) << 32)
            else:
                prec = L.FMT_PREC_DEFAULT if it[2] is None else min(it[2], L.FMT_PREC_DEFAULT - 1)
                words.append(ord(it[1]) | (prec << 16))
        rec = self.ctx._heap_put(words)
        direct = isinstance(arg, ListLit) and len(arg.elems) <= FORMAT_MAX_STACK_ARGS
        mode = L.FORMAT_ARGS_STACK if direct else L.FORMAT_ARGS_LIST
        self.push_const(ConstVal(T["INT"], rec | (mode << 32)))
        args = arg.elems if direct else [arg]
        for e in args:
            self.expr(e)
        self.emit("FN", a=L.FNS["FORMAT"], b=1 + len(args), delta=-len(args))

    # ---- SPIFFE (conditions/types/spiffe.go): ids and trust domains are strings of a validated shape (tags SPIFFE_ID /
    # SPIFFE_TD); a matcher is never a run-time value -- spiffeMatchX(arg).matchesID(x) compiles to one fused function
    _SPIFFE1 = {"spiffeID": "SPIFFE_ID", "spiffeTrustDomain": "SPIFFE_TD"}
    _SPIFFE_RECV = {"path": "SPIFFE_PATH", "trustDomain": "SPIFFE_TD_OF", "name": "SPIFFE_TD_NAME"}
    _SPIFFE_MATCH = {"spiffeMatchExact": "SPIFFE_MATCH_EXACT", "spiffeMatchOneOf": "SPIFFE_MATCH_ONEOF", "spiffeMatchTrustDomain": "SPIFFE_MATCH_TD"}

    def _fn(self, name, argc):
        self.emit("FN", a=L.FNS[name], b=argc, delta=1 - argc)

    def _spiffe_call(self, n: Call, fn, args) -> bool:
        if fn in self._SPIFFE1 and n.target is None and len(args) == 1:
            self.expr(args[0])
            self._fn(self._SPIFFE1[fn], 1)
            return True
        if fn in self._SPIFFE_RECV and n.target is not None and len(args) == 1:
            self.expr(args[0])
            self._fn(self._SPIFFE_RECV[fn], 1)
            return True
        if fn == "id" and n.target is not None and len(args) == 1:      # spiffeTrustDomain(..).id(); id(x) of any other value is x
            self.expr(args[0])
            self._fn("SPIFFE_TD_ID", 1)
            return True
        if fn == "isMemberOf" and n.target is not None and len(args) == 2:
            self.expr(args[0])
            self.expr(args[1])
            self._fn("SPIFFE_MEMBER", 2)
            return True
        if fn == "matchesID" and n.target is not None and len(args) == 2:
            m = n.target
            if not (isinstance(m, Call) and m.target is None):
                raise Unsupported("matchesID on a matcher that is not built in place")
            if m.fn == "spiffeMatchAny" and not m.args:
                self.expr(args[1])
                self._fn("SPIFFE_MATCH_ANY", 1)
                return True
            if m.fn in self._SPIFFE_MATCH and len(m.args) == 1:
                a = m.args[0]
                if m.fn == "spiffeMatchOneOf" and isinstance(a, ListLit):
                    # a literal list of ids: spiffeID(e) elements are validated where they stand and travel as their id strings
                    for e in a.elems:
                        if isinstance(e, Call) and e.fn == "spiffeID" and e.target is None and len(e.args) == 1:
                            self.expr(e.args[0])
                            self._fn("SPIFFE_IDSTR", 1)
                        else:
                            self.expr(e)
                    self.emit("MKLIST", c=len(a.elems), delta=1 - len(a.elems))
                else:
                    self.expr(a)
                self.expr(args[1])
                self._fn(self._SPIFFE_MATCH[m.fn], 2)
                return True
            raise Unsupported("matchesID on a matcher that is not built in place")
        if fn in self._SPIFFE_MATCH or fn == "spiffeMatchAny":
            raise Unsupported("a SPIFFE matcher used as a value")
        return False

    # ---- hierarchy(s[, delim]) (conditions/types/hierarchy.go): never a run-time value -- the functions over
    # hierarchies compile to fused ops on the underlying strings
    def _hier(self, n):
        """-> (string expression, delimiter string id) if n is hierarchy(expr[, "delim"]), else None"""
        if not (isinstance(n, Call) and n.fn == "hierarchy" and n.target is None and len(n.args) in (1, 2)):
            return None
        delim = "."
        if len(n.args) == 2:
            d = n.args[1]
            if not (isinstance(d, Const) and isinstance(d.value, str) and d.value):
                raise Unsupported("hierarchy() with a non-constant or empty delimiter")
            delim = d.value
        if isinstance(n.args[0], MapLit):
            raise Unsupported("hierarchy() of a map")
        if isinstance(n.args[0], ListLit) or (isinstance(n.args[0], Macro) and n.args[0].name in ("map", "filter", "transformList")) or \
                (isinstance(n.args[0], Call) and n.args[0].fn in ("split", "except", "intersect", "sort", "slice", "flatten", "distinct")):
            # hierarchy(list of strings): the parts themselves -- joined on the device by U+001F, the delimiter the fused ops then split on
            if len(n.args) == 2:
                raise Unsupported("hierarchy(list, delimiter)")
            did = self.ctx.strings.intern("\x1f")
            if did > 0xFFFF:
                raise Unsupported("too many table strings for a hierarchy delimiter")
            return Call("@hier_join", None, [n.args[0]]), did
        did = self.ctx.strings.intern(delim)
        if did > 0xFFFF:
            raise Unsupported("too many table strings for a hierarchy delimiter")
        return n.args[0], did

    def _hier_ca(self, n):
        """-> ((s, ds), (t, dt)) if n is hierarchy(..).commonAncestors(hierarchy(..))"""
        if isinstance(n, Call) and n.fn == "commonAncestors" and n.target is not None and len(n.args) == 1:
            a, b = self._hier(n.target), self._hier(n.args[0])
            if a and b:
                return a, b
        return None

    def _hier_call(self, fn, args) -> bool:
        if fn in L.HIER_RELS and fn != "equals" and len(args) == 2:
            a, b = self._hier(args[0]), self._hier(args[1])
            if not (a and b):
                return False
            self.expr(a[0])
            self.expr(b[0])
            self.emit("HIER_REL", a=L.HIER_RELS[fn], b=a[1], c=b[1], delta=-1)
            return True
        if fn in ("_==_", "_!=_") and len(args) == 2:
            for x, y in ((args[0], args[1]), (args[1], args[0])):
                ca, hz = self._hier_ca(x), self._hier(y)
                if ca and hz:
                    self.expr(ca[0][0])
                    self.expr(ca[1][0])
                    self.expr(hz[0])
                    self.emit("HIER_CA", a=1, b=ca[0][1], c=ca[1][1] | (hz[1] << 16), delta=-2)
                    if fn == "_!=_":
                        self.emit("NOT")
                    return True
            a, b = self._hier(args[0]), self._hier(args[1])
            if a and b:
                self.expr(a[0])
                self.expr(b[0])
                self.emit("HIER_REL", a=L.HIER_RELS["equals"], b=a[1], c=b[1], delta=-1)
                if fn == "_!=_":
                    self.emit("NOT")
                return True
            return False
        if fn == "size" and len(args) == 1:
            ca = self._hier_ca(args[0])
            if ca:
                self.expr(ca[0][0])
                self.expr(ca[1][0])
                self.emit("HIER_CA", a=0, b=ca[0][1], c=ca[1][1], delta=-1)
                return True
            h = self._hier(args[0])
            if h:
                self.expr(h[0])
                self.emit("HIER_SIZE", b=h[1])
                return True
        return False

    def _macro(self, n: Macro):
        kinds = {"all": (L.LOOP_ALL, 1), "exists": (L.LOOP_EXISTS, 1), "exists_one": (L.LOOP_EXISTS_ONE, 1),
                 "all2": (L.LOOP_ALL, 2), "exists2": (L.LOOP_EXISTS, 2), "exists_one2": (L.LOOP_EXISTS_ONE, 2),
                 # collecting comprehensions: the result is built in the device's scratch arena
                 "map": (L.LOOP_MAP, 1), "filter": (L.LOOP_FILTER, 1), "transformList": (L.LOOP_MAP, 2),
                 "transformMap": (L.LOOP_TMAP, 2), "transformMapEntry": (L.LOOP_TENTRY, 2), "sortBy": (L.LOOP_SORTBY, 1)}
        if n.name == "bind":
            # cel.bind(x, init, body) (ext.Bindings): the expressions are pure, so the body with x replaced by init has the same
            # value (an init that fails and is never used harms nothing either way)
            return self.expr(expand_bind(n))
        if n.name not in kinds:
            raise Unsupported(f"macro `{n.name}`")
        kind, nv = kinds[n.name]
        depth = len(self.loop_vars)
        if depth >= L.MAX_LOOP_DEPTH:
            raise Unsupported("comprehension nesting too deep")
        self.ctx.max_loop_depth = max(self.ctx.max_loop_depth, depth + 1)
        base = depth * 2
        self.ctx.n_vars = max(self.ctx.n_vars, base + 2)
        self.expr(n.target)
        init = self.emit("LOOP_INIT", a=base, b=kind | (0x100 if nv == 2 else 0), delta=-1)
        frame = {n.vars[0]: base} if nv == 1 else {n.vars[0]: base, n.vars[1]: base + 1}
        self.loop_vars.append(frame)
        body = self.here()
        pred = None
        if len(n.args) == 2:          # map(x, pred, f) / transform*(k, v, pred, f): iterations whose predicate is false are skipped
            self.expr(n.args[0])
            pred = self.emit("LOOP_PRED", delta=-1)
        self.expr(n.args[-1])
        nxt = self.emit("LOOP_NEXT", a=base, b=kind | (0x100 if nv == 2 else 0), c=body, delta=-1)
        if pred is not None:
            self.patch(pred, "c", nxt)
        self.loop_vars.pop()
        self.sp += 1  # loop result
        self.patch(init, "c", self.here())

    # ---------------------------------------------------------------- entry
    def finish(self):
        self.emit("RET")
        return self.code


_FMT_VERBS = "sdfebxXo"
# list-literal elements FORMAT takes from the operand stack: with the clause record and the enclosing expression's operands
# they must fit the device's evaluation stack (layout.MAX_STACK = 16)
FORMAT_MAX_STACK_ARGS = L.MAX_STACK - 4


def parse_format(fmt: str):
    """Clauses of a format string as cel-go's ext.Strings reads them (restated by oracle #1, celeval._str_format):
    [("lit", text) | ("verb", verb, precision or None)], or None when a clause is malformed -- a lone `%` at the end, a
    precision with no verb after it, or a verb outside %s %d %f %e %b %x %X %o -- which makes every call an error."""
    items, lit = [], []
    i, n = 0, len(fmt)
    while i < n:
        ch = fmt[i]
        if ch != "%":
            lit.append(ch)
            i += 1
            continue
        i += 1
        if i >= n:
            return None
        if fmt[i] == "%":
            lit.append("%")
            i += 1
            continue
        prec = None
        if fmt[i] == ".":
            j = i + 1
            while j < n and fmt[j].isdigit():
                j += 1
            digits = fmt[i + 1:j]
            if not digits.isascii():
                raise Unsupported("format() clause with a precision in non-ASCII digits")
            prec = int(digits or "0")
            i = j
        if i >= n or fmt[i] not in _FMT_VERBS:
            return None
        if lit:
            items.append(("lit", "".join(lit)))
            lit = []
        items.append(("verb", fmt[i], prec))
        i += 1
    if lit:
        items.append(("lit", "".join(lit)))
    return items


def _substitute(node, name, repl, repl_free):
    """`node` with every free occurrence of the identifier `name` replaced by `repl`"""
    if isinstance(node, Ident):
        return repl if node.name == name else node
    if isinstance(node, Select):
        return Select(_substitute(node.operand, name, repl, repl_free), node.field, node.test_only)
    if isinstance(node, Call):
        return Call(node.fn, None if node.target is None else _substitute(node.target, name, repl, repl_free),
                    [_substitute(a, name, repl, repl_free) for a in node.args])
    if isinstance(node, ListLit):
        return ListLit([_substitute(e, name, repl, repl_free) for e in node.elems])
    if isinstance(node, MapLit):
        return MapLit([(_substitute(k, name, repl, repl_free), _substitute(v, name, repl, repl_free)) for k, v in node.entries])
    if isinstance(node, Macro):
        target = _substitute(node.target, name, repl, repl_free)
        if name in node.vars:
            return Macro(node.name, target, node.vars, node.args)        # shadowed inside
        if repl_free & set(node.vars) and any(isinstance(z, Ident) and z.name == name for a in node.args for z in walk_nodes(a)):
            raise Unsupported("cel.bind: the bound expression mentions a name that a comprehension inside the body redefines")
        return Macro(node.name, target, node.vars, [_substitute(a, name, repl, repl_free) for a in node.args])
    return node


def expand_bind(n: Macro):
    free = {z.name for z in walk_nodes(n.target) if isinstance(z, Ident)}
    return _substitute(n.args[0], n.vars[0], n.target, free)


class FlatCompiler:
    """Lowers a condition to disjunctive normal form over simple *terms* (layout.FLAT_DNF) for the kernels'
    call-free fast path.

    A condition leaf only asks "is the result BOOL true" (ruletable.go:1425-1441).  With
    T(e) = "e is BOOL true" and F(e) = "e is BOOL false", cel-go's error-absorbing logic gives
        T(a && b) = T(a) & T(b)      F(a && b) = F(a) | F(b)
        T(a || b) = T(a) | T(b)      F(a || b) = F(a) & F(b)
        T(!a)     = F(a)             F(!a)     = T(a)
        T(c ? a : b) = T(c) & T(a) | F(c) & T(b)        F(c ? a : b) = T(c) & F(a) | F(c) & F(b)
    so any expression over term leaves has an exact DNF over the literals T(term) / F(term); all / any of such
    leaves compose the same way and a top-level `none` is a final negation.  A term is a compare, `in`, string
    predicate, set predicate or has() whose operands are attribute slots, constants, P.id, a constant-index list
    element or size(slot).  `list.exists(x, x == e)` is `e in list`, `list.all(x, x != e)` is F(e in list)
    (only as positive literals: with an erroring `e` the comprehension and `in` differ in *which* non-true value
    they produce)."""

    MAX_TERMS = L.FLAT_MAX_TERMS

    def __init__(self, pc: "ProgramCompiler"):
        self.pc = pc

    # ---- operands
    def operand(self, n: Node):
        """-> (kind, value, aux) or None"""
        pc = self.pc
        if isinstance(n, Call) and n.fn == "size" and len(([n.target] if n.target is not None else []) + n.args) == 1:
            arg = n.target if n.target is not None else n.args[0]
            s = pc._simple(arg)
            if s is not None and s[0] == "slot":
                return (L.OPK["SLOT_SIZE"], pc._slot_ix(s[1]), 0)
            return None
        if isinstance(n, Call) and n.fn == "_[_]" and n.target is None and isinstance(n.args[1], Const) \
                and isinstance(n.args[1].value, int) and not isinstance(n.args[1].value, bool):
            s = pc._simple(n.args[0])
            idx = int(n.args[1].value)
            if s is not None and s[0] == "slot" and 0 <= idx < 0xFFFF:
                return (L.OPK["SLOT_ELEM"], pc._slot_ix(s[1]), idx)
            return None
        s = pc._simple(n)
        if s is None:
            return None
        if s[0] == "slot":
            return (L.OPK["SLOT"], pc._slot_ix(s[1]), 0)
        if s[0] == "pid":
            pc.ctx.uses_pid = True
            return (L.OPK["PID"], 0, 0)
        cix = pc._const_ix(s[1])
        if const_v64(pc.ctx, pc.ctx.consts[cix]) == L.FLAT_NOT_FAST:
            return None
        return (L.OPK["CONST"], cix, 0)

    @staticmethod
    def mk(op, x, y, ci=0):
        return {"op": L.TERM_OPS[op], "ci": ci, "x": x, "y": y if y is not None else (L.OPK["CONST"], 0, 0)}

    def term(self, n: Node):
        """-> term dict (value = the expression itself) or None"""
        if isinstance(n, Select) and n.test_only:
            try:
                st = self.pc._static(Select(n.operand, n.field))
            except Unsupported:
                return None
            if st is None or st.kind != "slot" or len(st.path) <= 2:
                return None
            return self.mk("HAS", (L.OPK["SLOT"], self.pc._slot_ix(st.path), 0), None)
        if isinstance(n, Call):
            args = ([n.target] if n.target is not None else []) + n.args
            if n.target is None and len(args) == 2 and n.fn in L.CMP_INDEX and n.fn != "_!=_":
                x, y = self.operand(args[0]), self.operand(args[1])
                if x is None or y is None:
                    return None
                return self.mk("CMP", x, y, L.CMP_INDEX[n.fn])
            if n.target is None and len(args) == 2 and n.fn == "@in":
                x, y = self.operand(args[0]), self.operand(args[1])
                if x is None or y is None or x[0] == L.OPK["SLOT_SIZE"] or y[0] not in (L.OPK["SLOT"], L.OPK["CONST"]):
                    return None
                return self.mk("IN", x, y)
            str2 = {"startsWith": "STARTS", "endsWith": "ENDS", "contains": "CONTAINS"}
            set2 = {"hasIntersection": "INTERSECTS", "has_intersection": "INTERSECTS", "isSubset": "SUBSET", "is_subset": "SUBSET"}
            if len(args) == 2 and (n.fn in str2 or n.fn in set2):
                x, y = self.operand(args[0]), self.operand(args[1])
                ok = (L.OPK["SLOT"], L.OPK["CONST"], L.OPK["PID"], L.OPK["SLOT_ELEM"]) if n.fn in str2 else (L.OPK["SLOT"], L.OPK["CONST"])
                if x is None or y is None or x[0] not in ok or y[0] not in ok:
                    return None
                return self.mk(str2.get(n.fn) or set2[n.fn], x, y)
        # a bare boolean attribute / constant: true <=> value == true, false <=> value == false
        if isinstance(n, (Select, Call, Ident, Const)):
            x = self.operand(n)
            if x is not None and x[0] in (L.OPK["SLOT"], L.OPK["SLOT_ELEM"]):
                return None   # a non-bool value would be an *error* as a logical operand but `== true` is false
        return None

    # ---- DNF: list of groups, each a list of (term, lit_false)
    def lit(self, n: Node, want_false: bool):
        if isinstance(n, Macro) and n.name == "bind":
            n = expand_bind(n)
        if isinstance(n, Call) and n.target is None:
            if n.fn == "!_" and len(n.args) == 1:
                return self.lit(n.args[0], not want_false)
            if n.fn in ("_&&_", "_||_") and len(n.args) == 2:
                a, b = self.lit(n.args[0], want_false), self.lit(n.args[1], want_false)
                if a is None or b is None:
                    return None
                conj = (n.fn == "_&&_") != want_false      # T(a&&b), F(a||b) are conjunctions
                return self._and(a, b) if conj else self._or(a, b)
            if n.fn == "_!=_" and len(n.args) == 2:
                return self.lit(Call("_==_", None, n.args), not want_false)
            if n.fn == "_?_:_" and len(n.args) == 3:
                ct, cf = self.lit(n.args[0], False), self.lit(n.args[0], True)
                a, b = self.lit(n.args[1], want_false), self.lit(n.args[2], want_false)
                if None in (ct, cf, a, b):
                    return None
                l, r = self._and(ct, a), self._and(cf, b)
                return None if l is None or r is None else self._or(l, r)
        if isinstance(n, Macro) and not want_false and len(n.vars) == 1 and len(n.args) == 1 and n.name in ("exists", "all"):
            body, var = n.args[0], n.vars[0]
            want_fn = "_==_" if n.name == "exists" else "_!=_"
            if isinstance(body, Call) and body.target is None and body.fn == want_fn and len(body.args) == 2:
                for a, o in ((body.args[0], body.args[1]), (body.args[1], body.args[0])):
                    if isinstance(a, Ident) and a.name == var and not any(isinstance(z, Ident) and z.name == var for z in walk_nodes(o)):
                        return self.lit(Call("@in", None, [o, n.target]), n.name == "all")
            return None
        t = self.term(n)
        if t is None:
            return None
        return [[(t, want_false)]]

    def _or(self, a, b):
        r = a + b
        return r if sum(len(g) for g in r) <= self.MAX_TERMS else None

    def _and(self, a, b):
        r = [ga + gb for ga in a for gb in b]
        return r if sum(len(g) for g in r) <= self.MAX_TERMS else None

    def cond(self, c: Cond):
        """-> (negate, dnf) or None"""
        if c.op == "expr":
            d = self.lit(c.expr.ast, False)
            return None if d is None else (0, d)
        if not c.children:
            return None
        subs = []
        for ch in c.children:
            r = self.cond(ch)
            if r is None or r[0]:
                return None
            subs.append(r[1])
        d = subs[0]
        for x in subs[1:]:
            d = self._and(d, x) if c.op == "all" else self._or(d, x)
            if d is None:
                return None
        return (1 if c.op == "none" else 0, d)


def walk_nodes(n):
    from ..cel.ast import walk
    return walk(n)


def compile_flat(ctx: TableBuilderCtx, cond: Cond, params: Params | None):
    """-> (negate, [term words...]) if the condition has a flat (DNF) fast form, else None.
    Each term is 16 bytes, returned as two instruction tuples (op, a, b, c) so it fits the CODE section."""
    pc = ProgramCompiler(ctx, params)
    try:
        r = FlatCompiler(pc).cond(cond)
    except Unsupported:
        return None
    if r is None:
        return None
    negate, dnf = r
    n_terms = sum(len(g) for g in dnf)
    if not (1 <= n_terms <= L.FLAT_MAX_TERMS):
        return None
    words = []
    for g in dnf:
        for j, (t, lit_false) in enumerate(g):
            t = _specialize_term(ctx, t)
            flags = (t["ci"] & L.TERM_CI_MASK) | (L.TERM_LIT_F if lit_false else 0) | (L.TERM_GROUP_END if j == len(g) - 1 else 0)
            (xk, xv, xa), (yk, yv, ya) = t["x"], t["y"]
            # {u8 op; u8 flags; u8 xk; u8 yk; u32 x} {u32 y; u16 xa; u16 ya}  as two (op, a, b, c) instruction slots
            words.append([t["op"], flags, xk | (yk << 8), xv])
            words.append([yv & 0xFF, (yv >> 8) & 0xFF, (yv >> 16) & 0xFFFF, xa | (ya << 16)])
    return negate, n_terms, words


def _v64_tag(bits: int) -> int:
    top = bits >> 48
    return top & 0xF if (top & 0xFFF0) == 0xFFF0 else 0


def _specialize_term(ctx: TableBuilderCtx, t: dict) -> dict:
    """CMP / IN terms whose operand kinds are (slot | scalar constant | P.id) get a shape-specific opcode: the device
    then runs straight-line code for the shape instead of decoding operand kinds and value classes per request."""
    S, C, P = L.OPK["SLOT"], L.OPK["CONST"], L.OPK["PID"]
    op, ci, x, y = t["op"], t["ci"], t["x"], t["y"]

    def ctag(o):
        return _v64_tag(const_v64(ctx, ctx.consts[o[1]])) if o[0] == C else -1

    def scalar_list(o):   # constant list whose elements are all double / null / bool / string
        if o[0] != C or ctag(o) != L.V64_LIST:
            return False
        off = ctx.consts[o[1]].bits
        n = ctx.theap[off]
        return all(_v64_tag(e) <= L.V64_STRING for e in ctx.theap[off + 1: off + 1 + n])

    new = None
    if op == L.TERM_OPS["CMP"] and ci == 0:
        if x[0] != S and y[0] == S:
            x, y = y, x                       # equality is symmetric
        if x[0] == S and y[0] == S:
            new = "EQ_SS"
        elif x[0] == S and y[0] == C and 0 <= ctag(y) <= L.V64_STRING:
            new = "EQ_SC"
        elif x[0] == S and y[0] == P:
            new = "EQ_SP"
    elif op == L.TERM_OPS["CMP"] and ci in (2, 3, 4, 5):
        if x[0] == C and y[0] == S:
            x, y, ci = y, x, {2: 4, 3: 5, 4: 2, 5: 3}[ci]   # c < s  <=>  s > c
        if x[0] == S and y[0] == S:
            new = "ORD_SS"
        elif x[0] == S and y[0] == C and ctag(y) == 0:
            new = "ORD_SC"
    elif op == L.TERM_OPS["IN"]:
        if x[0] == S and scalar_list(y):
            new = "IN_SC"
        elif x[0] == C and 0 <= ctag(x) <= L.V64_STRING and y[0] == S:
            new = "IN_CS"
        elif x[0] == S and y[0] == S:
            new = "IN_SS"
    if new is None:
        return t
    return {"op": L.TERM_OPS[new], "ci": ci, "x": x, "y": y}


def const_v64(ctx: TableBuilderCtx, cv: ConstVal) -> int:
    """8-byte fast form of a constant for the flat path (layout.FLAT_NOT_FAST if it has none).
    INT constants become doubles: cel-go compares int with double by converting the int
    (types/compare.go compareDoubleInt), so this is exact for comparisons against attribute doubles."""
    if cv.tag == T["NULL"]:
        return box(L.V64_NULL)
    if cv.tag == T["BOOL"]:
        return box(L.V64_BOOL, cv.bits)
    if cv.tag == T["STRING"]:
        return box(L.V64_STRING, cv.bits)
    if cv.tag == T["DOUBLE"]:
        return cv.bits
    if cv.tag == T["INT"]:
        v = cv.bits - (1 << 64) if cv.bits >> 63 else cv.bits
        return f64_bits(float(v))
    if cv.tag == T["LIST"]:
        return box(L.V64_LIST, cv.bits)
    if cv.tag == T["MAP"]:
        return box(L.V64_MAP, cv.bits)
    return L.FLAT_NOT_FAST


def compile_condition(ctx: TableBuilderCtx, cond: Cond, params: Params | None) -> list:
    """Condition tree -> instruction list [[op, a, b, c], ...] leaving a plain BOOL."""
    pc = ProgramCompiler(ctx, params)
    pc.compile_cond(cond)
    assert pc.sp == 1, pc.sp
    return pc.finish()


def compile_value(ctx: TableBuilderCtx, expr, params: Params | None) -> list:
    """Expression -> instruction list leaving its VALUE (a rule output): the condition compiler's path without TO_COND."""
    pc = ProgramCompiler(ctx, params)
    pc.stack_limit = L.OUT_MAX_STACK
    pc.expr(expr.ast)
    assert pc.sp == 1, pc.sp
    return pc.finish()
