"""Tree-walking CEL evaluator with cel-go semantics -- TEST INFRASTRUCTURE (oracle).

Restates the behaviour of ``github.com/google/cel-go v0.27.0`` (go.mod:45 of the
reference; NOT vendored in the reference tree) as configured by
``conditions.StdEnv`` (internal/conditions/cel.go:62-75): standard CEL,
heterogeneous equality, CrossTypeNumericComparisons, ext.Strings / Lists /
Bindings / Encoders / Math / TwoVarComprehensions, plus the Cerbos library
(internal/conditions/cerbos_lib.go:38-135, 287-484) and the hierarchy type
(internal/conditions/types/hierarchy.go:146-410).

Errors are Python exceptions (CelError); ``&&``/``||``/all/exists absorb them the
way cel-go's error-as-value evaluation does.  Pinned by the reference goldens in
tests/golden/cel_eval.json and tests/golden/cerbos_lib_test.json.
"""
from __future__ import annotations

import base64 as _b64
import datetime as _dt
import ipaddress
import math
import os
import re
import struct

from cerbos_b200.cel.ast import Call, Const, Ident, ListLit, Macro, MapLit, Select, UInt

INT64_MIN = -(1 << 63)
INT64_MAX = (1 << 63) - 1
UINT64_MAX = (1 << 64) - 1

# time.Time range accepted by cel-go timestamps: 0001-01-01T00:00:00Z .. 9999-12-31T23:59:59.999999999Z
_MIN_TS_S = -62135596800
_MAX_TS_S = 253402300799


class CelError(Exception):
    """A CEL error value (cel-go types.Err)."""


def no_overload(fn="", *args):
    return CelError(f"no such overload: {fn}({', '.join(type_name(a) for a in args)})")


# ----------------------------------------------------------------------------- values

class Timestamp:
    __slots__ = ("ns",)

    def __init__(self, ns: int):
        s = ns // 1_000_000_000
        if s < _MIN_TS_S or s > _MAX_TS_S:
            raise CelError("timestamp out of range")
        self.ns = ns

    def __repr__(self):
        return f"Timestamp({self.ns})"

    def __eq__(self, o):
        return isinstance(o, Timestamp) and o.ns == self.ns

    def __hash__(self):
        return hash(("ts", self.ns))


class Duration:
    __slots__ = ("ns",)

    def __init__(self, ns: int):
        if ns < INT64_MIN or ns > INT64_MAX:
            raise CelError("duration out of range")
        self.ns = ns

    def __repr__(self):
        return f"Duration({self.ns})"

    def __eq__(self, o):
        return isinstance(o, Duration) and o.ns == self.ns

    def __hash__(self):
        return hash(("dur", self.ns))


class CelType:
    __slots__ = ("name",)

    def __init__(self, name):
        self.name = name

    def __repr__(self):
        return f"type({self.name})"


class Hierarchy:
    __slots__ = ("parts",)

    def __init__(self, parts):
        self.parts = tuple(parts)

    def __repr__(self):
        return f"hierarchy({'.'.join(self.parts)})"


# ---- SPIFFE types (internal/conditions/types/spiffe.go over github.com/spiffe/go-spiffe/v2 v2.x, go.mod -- a third-party
# dependency outside the reference tree: its spiffeid.FromString / TrustDomainFromString / ValidatePath rules are
# restated here from the library's published source and pinned by the reference's TestCerbosLib rows and cel_eval goldens)
_TD_CHARS = set("abcdefghijklmnopqrstuvwxyz0123456789-._")
_SEG_CHARS = _TD_CHARS | set("ABCDEFGHIJKLMNOPQRSTUVWXYZ")


def spiffe_parse_id(s: str):
    """spiffeid.FromString -> (id string, index where the path starts) or raises CelError"""
    if s == "":
        raise CelError("failed to parse SPIFFE ID: cannot be empty")
    if not s.startswith("spiffe://"):
        raise CelError("failed to parse SPIFFE ID: scheme is missing or invalid")
    i = 9
    while i < len(s) and s[i] != "/":
        if s[i] not in _TD_CHARS:
            raise CelError("failed to parse SPIFFE ID: trust domain characters are limited to lowercase letters, numbers, dots, dashes, and underscores")
        i += 1
    if i == 9:
        raise CelError("failed to parse SPIFFE ID: trust domain is missing")
    path = s[i:]
    if path:                                   # spiffeid.ValidatePath
        for seg in path[1:].split("/"):
            if seg == "":
                raise CelError("failed to parse SPIFFE ID: path cannot contain empty segments / have a trailing slash")
            if seg in (".", ".."):
                raise CelError("failed to parse SPIFFE ID: path cannot contain dot segments")
            if any(ch not in _SEG_CHARS for ch in seg):
                raise CelError("failed to parse SPIFFE ID: path segment characters are limited to letters, numbers, dots, dashes, and underscores")
    return s, i


def spiffe_parse_td(s: str) -> str:
    """spiffeid.TrustDomainFromString -> trust domain name"""
    if s == "":
        raise CelError("failed to parse SPIFFE trust domain: trust domain is missing")
    if ":/" in s:
        sid, i = spiffe_parse_id(s)
        return sid[9:i]
    if any(ch not in _TD_CHARS for ch in s):
        raise CelError("failed to parse SPIFFE trust domain: trust domain characters are limited to lowercase letters, numbers, dots, dashes, and underscores")
    return s


class SpiffeID:
    __slots__ = ("id", "pathidx")

    def __init__(self, s):
        self.id, self.pathidx = spiffe_parse_id(s)

    @property
    def td(self):
        return self.id[9:self.pathidx]


class SpiffeTD:
    __slots__ = ("name",)

    def __init__(self, name):
        self.name = name


class SpiffeMatcher:
    __slots__ = ("kind", "arg")     # "any" | "exact" (id string) | "oneof" (set of id strings) | "td" (name)

    def __init__(self, kind, arg=None):
        self.kind, self.arg = kind, arg

    def matches(self, sid: SpiffeID) -> bool:
        if self.kind == "any":
            return True
        if self.kind == "exact":
            return sid.id == self.arg
        if self.kind == "oneof":
            return sid.id in self.arg
        return sid.td == self.arg


class CelMap:
    """Insertion-ordered CEL map with type-aware key lookup."""
    __slots__ = ("keys", "vals", "_sidx")

    def __init__(self, items=()):
        self.keys = []
        self.vals = []
        self._sidx = {}
        for k, v in items:
            self.put(k, v)

    def put(self, k, v):
        i = self._index(k)
        if i is not None:
            self.vals[i] = v
            return
        if type(k) is str:
            self._sidx[k] = len(self.keys)
        self.keys.append(k)
        self.vals.append(v)

    def _index(self, k):
        if type(k) is str:
            return self._sidx.get(k)
        for i, kk in enumerate(self.keys):
            if type(kk) is not str and cel_equal(kk, k):
                return i
        return None

    def find(self, k):
        """Returns (found, value)."""
        i = self._index(k)
        if i is None:
            return False, None
        return True, self.vals[i]

    def __len__(self):
        return len(self.keys)

    def items(self):
        return zip(self.keys, self.vals)

    def __repr__(self):
        return "CelMap{" + ", ".join(f"{k!r}: {v!r}" for k, v in self.items()) + "}"


class Msg:
    """A protobuf message value (Request, Request.Principal, Request.Resource,
    AuxData, Runtime -- api/public/cerbos/engine/v1/engine.proto)."""
    __slots__ = ("type_name", "fields", "aliases")

    def __init__(self, type_name, fields, aliases=None):
        self.type_name = type_name
        self.fields = fields  # name -> value (always populated with defaults)
        self.aliases = aliases or {}

    def resolve(self, name):
        name = self.aliases.get(name, name)
        if name not in self.fields:
            raise CelError(f"no such field '{name}'")
        return name

    def get(self, name):
        return self.fields[self.resolve(name)]

    def has(self, name):
        v = self.fields[self.resolve(name)]
        # proto3 presence: scalars are "set" when non-default, repeated/map when non-empty,
        # sub-messages when present.
        if v is None:
            return False
        if isinstance(v, Msg):
            return not getattr(v, "_absent", False) and v.type_name != "<absent>"
        if isinstance(v, (str, bytes, list, CelMap)):
            return len(v) > 0
        if isinstance(v, bool):
            return v
        if isinstance(v, (int, float)):
            return v != 0
        return True


class AbsentMsg(Msg):
    """An unset sub-message field: selects behave like the default instance, has() is false."""
    __slots__ = ()


def type_name(v) -> str:
    if v is None:
        return "null_type"
    if isinstance(v, bool):
        return "bool"
    if isinstance(v, UInt):
        return "uint"
    if isinstance(v, int):
        return "int"
    if isinstance(v, float):
        return "double"
    if isinstance(v, str):
        return "string"
    if isinstance(v, bytes):
        return "bytes"
    if isinstance(v, list):
        return "list"
    if isinstance(v, CelMap):
        return "map"
    if isinstance(v, Timestamp):
        return "google.protobuf.Timestamp"
    if isinstance(v, Duration):
        return "google.protobuf.Duration"
    if isinstance(v, CelType):
        return "type"
    if isinstance(v, Hierarchy):
        return "cerbos.lib.hierarchy"
    if isinstance(v, Msg):
        return v.type_name
    return type(v).__name__


def from_json(v):
    """google.protobuf.Value -> CEL value (numbers are always doubles)."""
    if v is None or isinstance(v, (bool, str)):
        return v
    if isinstance(v, (int, float)):
        return float(v)
    if isinstance(v, (list, tuple)):
        return [from_json(x) for x in v]
    if isinstance(v, dict):
        return CelMap((str(k), from_json(x)) for k, x in v.items())
    raise TypeError(f"not a JSON value: {type(v)}")


# ----------------------------------------------------------------------------- numerics

def is_num(v):
    return isinstance(v, (int, float)) and not isinstance(v, bool)


def _cmp(a, b):
    return -1 if a < b else (1 if a > b else 0)


def num_compare(a, b, for_equality=False):
    """cel-go compare across int/uint/double. Returns -1/0/1, or None for NaN when
    for_equality; raises for NaN ordering."""
    fa, fb = isinstance(a, float), isinstance(b, float)
    if fa or fb:
        x = a if fa else None
        y = b if fb else None
        if (fa and math.isnan(a)) or (fb and math.isnan(b)):
            if for_equality:
                return None
            raise CelError("NaN values cannot be ordered")
        if fa and fb:
            return _cmp(a, b)
        # mixed: cel-go compareDoubleInt / compareDoubleUint (types/compare.go)
        if fa:
            d, i, sign = a, b, 1
        else:
            d, i, sign = b, a, -1
        if isinstance(i, UInt):
            if d < 0:
                r = -1
            elif d > float(UINT64_MAX):
                r = 1
            else:
                r = _cmp(d, float(i))
        else:
            if d < float(INT64_MIN):
                r = -1
            elif d > float(INT64_MAX):
                r = 1
            else:
                r = _cmp(d, float(i))
        return r * sign
    return _cmp(int(a), int(b))


def cel_equal(a, b) -> bool:
    """Heterogeneous equality (cel-go types.Equal)."""
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, bool) or isinstance(b, bool):
        return isinstance(a, bool) and isinstance(b, bool) and a == b
    if is_num(a):
        if not is_num(b):
            return False
        return num_compare(a, b, for_equality=True) == 0
    if isinstance(a, str):
        return isinstance(b, str) and a == b
    if isinstance(a, bytes):
        return isinstance(b, bytes) and a == b
    if isinstance(a, list):
        if not isinstance(b, list) or len(a) != len(b):
            return False
        return all(cel_equal(x, y) for x, y in zip(a, b))
    if isinstance(a, CelMap):
        if not isinstance(b, CelMap) or len(a) != len(b):
            return False
        for k, v in a.items():
            found, ov = b.find(k)
            if not found or not cel_equal(v, ov):
                return False
        return True
    if isinstance(a, Timestamp):
        return isinstance(b, Timestamp) and a.ns == b.ns
    if isinstance(a, Duration):
        return isinstance(b, Duration) and a.ns == b.ns
    if isinstance(a, CelType):
        return isinstance(b, CelType) and a.name == b.name
    if isinstance(a, Hierarchy):
        if not isinstance(b, Hierarchy):
            raise no_overload("_==_", a, b)
        return a.parts == b.parts
    if isinstance(a, SpiffeID):                      # spiffe.go:346-360
        if isinstance(b, SpiffeID):
            return a.id == b.id
        if isinstance(b, str):
            return a.id == b
        raise no_overload("_==_", a, b)
    if isinstance(a, SpiffeTD):                      # spiffe.go:443-461: a string that is no trust domain is simply unequal
        if isinstance(b, SpiffeTD):
            return a.name == b.name
        if isinstance(b, str):
            try:
                return spiffe_parse_td(b) == a.name
            except CelError:
                return False
        raise no_overload("_==_", a, b)
    if isinstance(a, SpiffeMatcher):                 # spiffe.go:538-540
        return False
    if isinstance(a, Msg):
        return isinstance(b, Msg) and a.type_name == b.type_name and all(
            cel_equal(a.fields[k], b.fields[k]) for k in a.fields)
    return False


def cel_compare(a, b, op):
    """Ordering for < <= > >= ; raises no_overload for unsupported pairs."""
    if isinstance(a, bool) or isinstance(b, bool):
        if isinstance(a, bool) and isinstance(b, bool):
            return _cmp(int(a), int(b))
        raise no_overload(op, a, b)
    if is_num(a) and is_num(b):
        return num_compare(a, b)
    if isinstance(a, str) and isinstance(b, str):
        return _cmp(a.encode("utf-8"), b.encode("utf-8"))
    if isinstance(a, bytes) and isinstance(b, bytes):
        return _cmp(a, b)
    if isinstance(a, Timestamp) and isinstance(b, Timestamp):
        return _cmp(a.ns, b.ns)
    if isinstance(a, Duration) and isinstance(b, Duration):
        return _cmp(a.ns, b.ns)
    raise no_overload(op, a, b)


def _chk_int(v):
    if v < INT64_MIN or v > INT64_MAX:
        raise CelError("integer overflow")
    return v


def _chk_uint(v):
    if v < 0 or v > UINT64_MAX:
        raise CelError("unsigned integer overflow")
    return UInt(v)


def _is_int(v):
    return isinstance(v, int) and not isinstance(v, (bool, UInt))


def _go_div(a, b):
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def _go_mod(a, b):
    return a - b * _go_div(a, b)


def _fdiv(a: float, b: float) -> float:
    if b == 0.0:
        if a == 0.0 or math.isnan(a):
            return math.nan
        neg = (math.copysign(1.0, a) < 0) != (math.copysign(1.0, b) < 0)
        return -math.inf if neg else math.inf
    return a / b


def op_add(a, b):
    if _is_int(a) and _is_int(b):
        return _chk_int(a + b)
    if isinstance(a, UInt) and isinstance(b, UInt):
        return _chk_uint(int(a) + int(b))
    if isinstance(a, float) and isinstance(b, float):
        return a + b
    if isinstance(a, str) and isinstance(b, str):
        return a + b
    if isinstance(a, bytes) and isinstance(b, bytes):
        return a + b
    if isinstance(a, list) and isinstance(b, list):
        return a + b
    if isinstance(a, Timestamp) and isinstance(b, Duration):
        return Timestamp(a.ns + b.ns)
    if isinstance(a, Duration) and isinstance(b, Timestamp):
        return Timestamp(a.ns + b.ns)
    if isinstance(a, Duration) and isinstance(b, Duration):
        return Duration(a.ns + b.ns)
    raise no_overload("_+_", a, b)


def op_sub(a, b):
    if _is_int(a) and _is_int(b):
        return _chk_int(a - b)
    if isinstance(a, UInt) and isinstance(b, UInt):
        return _chk_uint(int(a) - int(b))
    if isinstance(a, float) and isinstance(b, float):
        return a - b
    if isinstance(a, Timestamp) and isinstance(b, Timestamp):
        return Duration(a.ns - b.ns)
    if isinstance(a, Timestamp) and isinstance(b, Duration):
        return Timestamp(a.ns - b.ns)
    if isinstance(a, Duration) and isinstance(b, Duration):
        return Duration(a.ns - b.ns)
    raise no_overload("_-_", a, b)


def op_mul(a, b):
    if _is_int(a) and _is_int(b):
        return _chk_int(a * b)
    if isinstance(a, UInt) and isinstance(b, UInt):
        return _chk_uint(int(a) * int(b))
    if isinstance(a, float) and isinstance(b, float):
        return a * b
    raise no_overload("_*_", a, b)


def op_div(a, b):
    if _is_int(a) and _is_int(b):
        if b == 0:
            raise CelError("division by zero")
        return _chk_int(_go_div(a, b))
    if isinstance(a, UInt) and isinstance(b, UInt):
        if b == 0:
            raise CelError("division by zero")
        return UInt(int(a) // int(b))
    if isinstance(a, float) and isinstance(b, float):
        return _fdiv(a, b)
    raise no_overload("_/_", a, b)


def op_mod(a, b):
    if _is_int(a) and _is_int(b):
        if b == 0:
            raise CelError("modulus by zero")
        if b == -1 and a == INT64_MIN:
            raise CelError("integer overflow")
        return _go_mod(a, b)
    if isinstance(a, UInt) and isinstance(b, UInt):
        if b == 0:
            raise CelError("modulus by zero")
        return UInt(int(a) % int(b))
    raise no_overload("_%_", a, b)


def op_neg(a):
    if _is_int(a):
        return _chk_int(-a)
    if isinstance(a, float):
        return -a
    if isinstance(a, Duration):
        return Duration(-a.ns)
    raise no_overload("-_", a)


# ----------------------------------------------------------------------------- time helpers

_RFC3339 = re.compile(
    r"\A([0-9]{4})-([0-9]{2})-([0-9]{2})T([0-9]{2}):([0-9]{2}):([0-9]{2})(?:[.,]([0-9]{1,9})[0-9]*)?(Z|[+-][0-9]{2}:[0-9]{2})\Z")


def _days_from_civil(y, m, d):
    y -= m <= 2
    era = (y if y >= 0 else y - 399) // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def _civil_from_days(z):
    z += 719468
    era = (z if z >= 0 else z - 146096) // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    y = yoe + era * 400
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + (3 if mp < 10 else -9)
    return y + (m <= 2), m, d


def parse_timestamp(s: str) -> Timestamp:
    m = _RFC3339.match(s)
    if not m:
        raise CelError(f"invalid timestamp {s!r}")
    y, mo, d, h, mi, sec = (int(m.group(i)) for i in range(1, 7))
    frac = m.group(7) or ""
    ns = int((frac + "000000000")[:9]) if frac else 0
    if not (1 <= mo <= 12 and 1 <= d <= 31 and h < 24 and mi < 60 and sec < 60):
        raise CelError(f"invalid timestamp {s!r}")
    dim = [31, 29 if (y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)) else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
    if d > dim[mo - 1]:
        raise CelError(f"invalid timestamp {s!r}")
    tz = m.group(8)
    off = 0
    if tz != "Z":
        # Go's time.Parse (which cel-go calls with time.RFC3339): 'T' and 'Z' literally, and a range test on the offset that
        # uses `>` ("some people do write offsets of 24 hours or 60 minutes")
        oh, om = int(tz[1:3]), int(tz[4:6])
        if oh > 24 or om > 60:
            raise CelError(f"invalid timestamp {s!r}")
        off = (oh * 3600 + om * 60) * (1 if tz[0] == "+" else -1)
    secs = _days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + sec - off
    if secs < -62135596800 or secs > 253402300799:      # cel-go (types/string.go): the instant within 0001-01-01 .. 9999-12-31
        raise CelError("timestamp overflow")
    return Timestamp(secs * 1_000_000_000 + ns)


_DUR_UNITS = {"ns": 1, "us": 1_000, "µs": 1_000, "μs": 1_000, "ms": 1_000_000,
              "s": 1_000_000_000, "m": 60_000_000_000, "h": 3_600_000_000_000}
_DUR_PART = re.compile(r"([0-9]*)(?:\.([0-9]*))?(ns|us|µs|μs|ms|s|m|h)")   # (ASCII digits only: \d would take any Unicode digit)


def parse_duration(s: str) -> Duration:
    """Go time.ParseDuration."""
    orig = s
    if not s:
        raise CelError("invalid duration")
    neg = False
    if s[0] in "+-":
        neg = s[0] == "-"
        s = s[1:]
    if s == "0":
        return Duration(0)
    if not s:
        raise CelError(f"invalid duration {orig!r}")
    total = 0
    pos = 0
    while pos < len(s):
        m = _DUR_PART.match(s, pos)
        if not m or (m.group(1) == "" and not m.group(2)):
            raise CelError(f"invalid duration {orig!r}")
        whole, frac, unit = m.group(1), m.group(2), m.group(3)
        if whole == "" and (frac is None or frac == ""):
            raise CelError(f"invalid duration {orig!r}")
        mult = _DUR_UNITS[unit]
        v = int(whole or "0") * mult
        if frac:
            v += int(frac) * mult // (10 ** len(frac))
        total += v
        pos = m.end()
    if neg:
        total = -total
    if total < INT64_MIN or total > INT64_MAX:
        raise CelError(f"invalid duration {orig!r}")
    return Duration(total)


_TZ_LINKS = None


def _tz_links():
    global _TZ_LINKS
    if _TZ_LINKS is None:
        _TZ_LINKS = {}
        p = "/usr/share/zoneinfo/tzdata.zi"
        if os.path.exists(p):
            with open(p, encoding="utf-8", errors="replace") as f:
                for line in f:
                    if line.startswith("L "):
                        parts = line.split()
                        if len(parts) >= 3:
                            _TZ_LINKS[parts[2]] = parts[1]
    return _TZ_LINKS


def _tz_offset_seconds(tz: str, unix_s: int) -> int:
    """Offset east of UTC for zone `tz` at instant unix_s (cel-go timeZone())."""
    if ":" in tz:
        ind = tz.index(":")
        try:
            hr = int(tz[:ind])
            mn = int(tz[ind + 1:])
        except ValueError:
            raise CelError(f"invalid timezone {tz!r}")
        offset = hr * 60 - mn if tz[0] == "-" else hr * 60 + mn
        return offset * 60
    if tz in ("UTC", ""):
        return 0
    import zoneinfo
    name = tz
    for _ in range(3):
        try:
            zi = zoneinfo.ZoneInfo(name)
            break
        except Exception:
            nxt = _tz_links().get(name)
            if nxt is None:
                raise CelError(f"unknown time zone {tz!r}")
            name = nxt
    else:
        raise CelError(f"unknown time zone {tz!r}")
    # zoneinfo only covers years 1..9999 via datetime
    try:
        dt = _dt.datetime.fromtimestamp(unix_s, tz=zi)
    except (OverflowError, OSError, ValueError):
        raise CelError("timestamp out of datetime range")
    return int(dt.utcoffset().total_seconds())


def _ts_fields(ts: Timestamp, tz):
    s, ns = divmod(ts.ns, 1_000_000_000)
    if tz is not None:
        if not isinstance(tz, str):
            raise no_overload("timestamp getter", ts, tz)
        s += _tz_offset_seconds(tz, s)
    days, rem = divmod(s, 86400)
    y, m, d = _civil_from_days(days)
    return dict(year=y, month=m, day=d, hour=rem // 3600, minute=rem % 3600 // 60, second=rem % 60,
                ms=ns // 1_000_000, dow=(days + 4) % 7, doy=days - _days_from_civil(y, 1, 1))


def format_timestamp(ts: Timestamp) -> str:
    f = _ts_fields(ts, None)
    ns = ts.ns % 1_000_000_000
    frac = ""
    if ns:
        frac = "." + f"{ns:09d}".rstrip("0")
    return f"{f['year']:04d}-{f['month']:02d}-{f['day']:02d}T{f['hour']:02d}:{f['minute']:02d}:{f['second']:02d}{frac}Z"


def format_double_f(d: float) -> str:
    """strconv.FormatFloat(d, 'f', -1, 64), which is how cel-go's Double converts to a string (types/double.go,
    ConvertToType): the shortest digits that round-trip, never an exponent.  (No vector of the reference holds a double
    outside 1e-4 .. 1e6, where this and the %g form below differ: that part is restated from the library, unpinned.)"""
    if math.isnan(d):
        return "NaN"
    if math.isinf(d):
        return "+Inf" if d > 0 else "-Inf"
    sign = "-" if math.copysign(1, d) < 0 else ""
    r = repr(abs(d))
    m, _, e = r.partition("e")
    ip, _, fp = m.partition(".")
    exp10 = int(e) if e else 0
    digits = ip + fp
    point = len(ip) + exp10                 # position of the decimal point within `digits`
    if point <= 0:
        digits, point = "0" * (1 - point) + digits, 1
    if point >= len(digits):
        digits += "0" * (point - len(digits))
    whole, frac = digits[:point].lstrip("0") or "0", digits[point:].rstrip("0")
    return sign + whole + ("." + frac if frac else "")


def format_double(d: float) -> str:
    """Go fmt %g / strconv.FormatFloat(d, 'g', -1, 64): shortest digits, %e form when
    the decimal exponent is < -4 or >= 6."""
    if math.isnan(d):
        return "NaN"
    if math.isinf(d):
        return "+Inf" if d > 0 else "-Inf"
    sign = "-" if math.copysign(1, d) < 0 else ""
    if d == 0:
        return sign + "0"
    mant, _, ex = f"{abs(d):.17e}".partition("e")
    # shortest round-trip digits
    r = repr(abs(d))
    if "e" in r:
        m2, e2 = r.split("e")
        exp10 = int(e2)
    else:
        m2, exp10 = r, 0
    ip, _, fp = m2.partition(".")
    alldig = ip + fp
    lead = len(alldig) - len(alldig.lstrip("0"))
    digits = alldig.lstrip("0").rstrip("0") or "0"
    # position of the decimal point relative to the first significant digit
    dp = len(ip) - lead + exp10
    x = dp - 1
    if x < -4 or x >= 6:
        m = digits[0] + ("." + digits[1:] if len(digits) > 1 else "")
        return f"{sign}{m}e{'+' if x >= 0 else '-'}{abs(x):02d}"
    if dp <= 0:
        return sign + "0." + "0" * (-dp) + digits
    if dp >= len(digits):
        return sign + digits + "0" * (dp - len(digits))
    return sign + digits[:dp] + "." + digits[dp:]


# ----------------------------------------------------------------------------- conversions

def conv_int(v):
    if _is_int(v):
        return v
    if isinstance(v, UInt):
        if v > INT64_MAX:
            raise CelError("integer overflow")
        return int(v)
    if isinstance(v, float):
        if math.isnan(v) or math.isinf(v) or v <= float(INT64_MIN) or v >= float(INT64_MAX):
            raise CelError("integer overflow")
        return int(v)
    if isinstance(v, str):
        if not re.fullmatch(r"[+-]?[0-9]+", v):
            raise CelError(f"cannot convert {v!r} to int")
        return _chk_int(int(v))
    if isinstance(v, Timestamp):
        return v.ns // 1_000_000_000
    if isinstance(v, Duration):
        return v.ns
    raise no_overload("int", v)


def conv_uint(v):
    if isinstance(v, UInt):
        return v
    if _is_int(v):
        if v < 0:
            raise CelError("unsigned integer overflow")
        return UInt(v)
    if isinstance(v, float):
        if math.isnan(v) or math.isinf(v) or v < 0 or v > float(UINT64_MAX):
            raise CelError("unsigned integer overflow")
        return _chk_uint(int(v))
    if isinstance(v, str):
        if not re.fullmatch(r"[0-9]+", v):     # strconv.ParseUint(s, 10, 64): "A sign prefix is not permitted"
            raise CelError(f"cannot convert {v!r} to uint")
        return _chk_uint(int(v))
    raise no_overload("uint", v)


def conv_double(v):
    if isinstance(v, bool):
        raise no_overload("double", v)
    if isinstance(v, float):
        return v
    if isinstance(v, int):
        return float(v)
    if isinstance(v, str):
        t = v.strip()
        if t != v or "_" in v:
            raise CelError(f"cannot convert {v!r} to double")
        try:
            return float(v)
        except ValueError:
            raise CelError(f"cannot convert {v!r} to double")
    raise no_overload("double", v)


def conv_string(v):
    if isinstance(v, str):
        return v
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, int):
        return str(int(v))
    if isinstance(v, float):
        return format_double_f(v)
    if isinstance(v, bytes):
        try:
            return v.decode("utf-8")
        except UnicodeDecodeError:
            raise CelError("invalid UTF-8 in bytes")
    if isinstance(v, Timestamp):
        return format_timestamp(v)
    if isinstance(v, Duration):
        s, ns = divmod(abs(v.ns), 1_000_000_000)
        sign = "-" if v.ns < 0 else ""
        if ns:
            return f"{sign}{s}.{f'{ns:09d}'.rstrip('0')}s"
        return f"{sign}{s}s"
    if isinstance(v, Hierarchy):
        return ".".join(v.parts)
    raise no_overload("string", v)


def conv_bool(v):
    if isinstance(v, bool):
        return v
    if isinstance(v, str):
        if v in ("1", "t", "T", "TRUE", "true", "True"):
            return True
        if v in ("0", "f", "F", "FALSE", "false", "False"):
            return False
        raise CelError(f"cannot convert {v!r} to bool")
    raise no_overload("bool", v)


def conv_bytes(v):
    if isinstance(v, bytes):
        return v
    if isinstance(v, str):
        return v.encode("utf-8")
    raise no_overload("bytes", v)


def conv_timestamp(v):
    if isinstance(v, Timestamp):
        return v
    if isinstance(v, str):
        return parse_timestamp(v)
    if _is_int(v):
        return Timestamp(v * 1_000_000_000)
    raise no_overload("timestamp", v)


def conv_duration(v):
    if isinstance(v, Duration):
        return v
    if isinstance(v, str):
        return parse_duration(v)
    if _is_int(v):
        return Duration(v)
    raise no_overload("duration", v)


# ----------------------------------------------------------------------------- strings ext

def _cps(s):
    return s  # Python str is already indexed by code point


def _need(cond, fn, *args):
    if not cond:
        raise no_overload(fn, *args)


_RE2_POSIX = {"alpha": "A-Za-z", "digit": "0-9", "alnum": "0-9A-Za-z", "upper": "A-Z", "lower": "a-z", "space": "\\t\\n\\v\\f\\r ",
              "punct": "!-/:-@\\[-`{-~", "xdigit": "0-9A-Fa-f", "word": "0-9A-Za-z_", "blank": "\\t ", "cntrl": "\\x00-\\x1f\\x7f",
              "print": " -~", "graph": "!-~", "ascii": "\\x00-\\x7f"}
_RE2_PERL = {"d": "0-9", "w": "0-9A-Za-z_", "s": "\\t\\n\\f\\r "}     # RE2's \s has no \v; all three are ASCII-only
_regex_cache: dict = {}


def _re2_to_python(p: str) -> str:
    r"""cel-go's `matches` is Go's regexp (RE2 syntax, regexp/syntax doc).  Python's `re` is the engine here, so the pattern
    is rewritten where the two differ: Perl classes are ASCII and \s lacks \v; `$` without (?m) is the end of the text only
    (Python's also matches before a final newline); \z; POSIX classes; \Q..\E; (?<name>; inline flags in the middle of a
    pattern scope to the end of their group; the U flag (greediness cannot change a yes / no answer).  What RE2 rejects --
    backreferences, lookaround, possessive / atomic forms, \Z, repeat counts over 1000 -- raises CelError like any
    invalid pattern; what `re` cannot express (\p{..}, \C, negated POSIX classes inside a larger class) raises too, and
    the product rejects those at table build, so they are never compared."""
    out, i, n = [], 0, len(p)
    multiline = False
    closers = [0]            # per open group: how many "(?flags:" wrappers to close with it
    first_atom = True

    def bad(why):
        return CelError(f"invalid regex {p!r}: {why}")

    while i < n:
        ch = p[i]
        if ch == "\\":
            if i + 1 >= n:
                raise bad("trailing backslash")
            e = p[i + 1]
            i += 2
            if e in "dws":
                out.append("[" + _RE2_PERL[e] + "]")
            elif e in "DWS":
                out.append("[^" + _RE2_PERL[e.lower()] + "]")
            elif e == "z":
                out.append("(?:\\Z)")
            elif e == "A":
                out.append("(?:\\A)")
            elif e == "b":       # ASCII word boundary (Python's \\b follows Unicode word characters)
                out.append("(?:(?<=[0-9A-Za-z_])(?![0-9A-Za-z_])|(?<![0-9A-Za-z_])(?=[0-9A-Za-z_]))")
            elif e == "B":
                out.append("(?:(?<=[0-9A-Za-z_])(?=[0-9A-Za-z_])|(?<![0-9A-Za-z_])(?![0-9A-Za-z_]))")
            elif e == "Z":
                raise bad("\\Z")
            elif e == "Q":
                j = p.find("\\E", i)
                lit = p[i:] if j < 0 else p[i:j]
                out.append(re.escape(lit))
                i = n if j < 0 else j + 2
            elif e in "pPC":
                raise bad("\\" + e + " is not supported by this oracle")
            elif e in "123456789":
                raise bad("backreference")
            elif e == "0":
                j = i
                while j < n and j < i + 2 and p[j] in "01234567":
                    j += 1
                out.append("\\x%02x" % int("0" + p[i:j], 8))
                i = j
            elif e == "x" and i < n and p[i] == "{":
                j = p.find("}", i)
                if j < 0:
                    raise bad("\\x{")
                out.append("\\U%08x" % int(p[i + 1:j], 16))
                i = j + 1
            else:
                out.append("\\" + e)
            first_atom = False
            continue
        if ch == "[":
            j = i + 1
            cls = ["["]
            if j < n and p[j] == "^":
                cls.append("^")
                j += 1
            if j < n and p[j] == "]":
                cls.append("\\]")
                j += 1
            while True:
                if j >= n:
                    raise bad("missing ]")
                c = p[j]
                if c == "]":
                    break
                if c == "[" and p.startswith("[:", j):
                    k = p.find(":]", j)
                    if k < 0:
                        raise bad("bad POSIX class")
                    name = p[j + 2:k]
                    if name.startswith("^") or name not in _RE2_POSIX:
                        raise bad(f"[:{name}:] is not supported by this oracle" if name.lstrip("^") in _RE2_POSIX else f"invalid character class [:{name}:]")
                    cls.append(_RE2_POSIX[name])
                    j = k + 2
                elif c == "\\":
                    if j + 1 >= n:
                        raise bad("trailing backslash")
                    e = p[j + 1]
                    if e in "dws":
                        cls.append(_RE2_PERL[e])
                    elif e in "DWSpPC":
                        raise bad("\\" + e + " inside a class is not supported by this oracle")
                    else:
                        cls.append("\\" + e)
                    j += 2
                else:
                    cls.append("\\" + c if c in "[&~|" else c)
                    j += 1
            cls.append("]")
            out.append("".join(cls))
            i = j + 1
            first_atom = False
            continue
        if ch == "(":
            if p.startswith("(?", i):
                k = i + 2
                if p.startswith("(?P<", i) or p.startswith("(?<", i) and not p.startswith("(?<=", i) and not p.startswith("(?<!", i):
                    j = p.find(">", i)
                    if j < 0:
                        raise bad("bad group name")
                    out.append("(?P<" + p[p.index("<", i) + 1:j] + ">")
                    closers.append(0)
                    i = j + 1
                    first_atom = False
                    continue
                while k < n and p[k] in "imsU-":
                    k += 1
                if k >= n or p[k] not in ":)":
                    raise bad("lookaround / atomic groups / comments are not RE2")
                flags = p[i + 2:k]
                on = flags.split("-")[0]
                if "m" in on:
                    multiline = True
                fl = flags.replace("U", "")
                if fl.endswith("-"):
                    fl = fl[:-1]
                if p[k] == ":":
                    out.append("(?" + fl + ":")
                    closers.append(0)
                elif fl:                       # (?flags): to the end of the enclosing group
                    if first_atom and len(closers) == 1 and "-" not in fl:
                        out.append("(?" + fl + ")")
                    else:
                        out.append("(?" + fl + ":")
                        closers[-1] += 1
                i = k + 1
                continue
            out.append("(")
            closers.append(0)
            i += 1
            first_atom = False
            continue
        if ch == ")":
            if len(closers) == 1:
                raise bad("unexpected )")
            out.append(")" * (closers.pop() + 1))
            i += 1
            continue
        if ch == "|" and closers[-1]:
            # an alternation inside a flag scope opened in the middle of a group: RE2's flags run to the end of the group,
            # across the |, which the scoped form here cannot say
            raise bad("inline flags before an alternation are not supported by this oracle")
        if ch == "$" or ch == "^":
            # (a group: Go lets a repetition operator follow an assertion -- `$?`, `^*` -- where `re` finds nothing to repeat)
            out.append("(?:^)" if ch == "^" else "(?:$)" if multiline else "(?:\\Z)")
            i += 1
            first_atom = False
            continue
        if ch in "*+?" or ch == "{":
            if ch == "{":
                m = re.match(r"\{(\d+)(,(\d*))?\}", p[i:])
                if not m:
                    out.append("\\{")
                    i += 1
                    continue
                if int(m.group(1)) > 1000 or (m.group(3) and int(m.group(3)) > 1000):
                    raise bad("repeat count over 1000")
                out.append(m.group(0))
                i += len(m.group(0))
            else:
                out.append(ch)
                i += 1
            if i < n and p[i] == "?":
                out.append("?")
                i += 1
            if i < n and (p[i] in "*+?" or re.match(r"\{\d+(,\d*)?\}", p[i:])):
                raise bad("nested repetition")
            continue
        out.append(ch)
        i += 1
        first_atom = False
    if len(closers) != 1:
        raise bad("missing )")
    out.append(")" * closers[0])
    return "".join(out)


def _regex(pattern: str):
    r = _regex_cache.get(pattern)
    if r is None:
        try:
            r = re.compile(_re2_to_python(pattern))
        except re.error as e:
            r = CelError(f"invalid regex {pattern!r}: {e}")
        except CelError as e:
            r = e
        _regex_cache[pattern] = r
    if isinstance(r, CelError):
        raise r
    return r


def _str_format(fmt: str, args: list) -> str:
    out = []
    i = 0
    ai = 0
    n = len(fmt)
    while i < n:
        c = fmt[i]
        if c != "%":
            out.append(c)
            i += 1
            continue
        i += 1
        if i >= n:
            raise CelError("unexpected end of format string")
        if fmt[i] == "%":
            out.append("%")
            i += 1
            continue
        prec = None
        if fmt[i] == ".":
            j = i + 1
            while j < n and fmt[j].isdigit():
                j += 1
            prec = int(fmt[i + 1:j] or "0")
            i = j
        verb = fmt[i]
        i += 1
        if ai >= len(args):
            raise CelError("index out of range in format")
        a = args[ai]
        ai += 1
        out.append(_fmt_verb(verb, prec, a))
    return "".join(out)


def _fmt_s(a):
    if a is None:
        return "null"
    if isinstance(a, list):
        return "[" + ", ".join(_fmt_s(x) for x in a) + "]"
    if isinstance(a, CelMap):
        items = sorted(((_fmt_s(k), _fmt_s(v)) for k, v in a.items()))
        return "{" + ", ".join(f"{k}: {v}" for k, v in items) + "}"
    if isinstance(a, CelType):
        return a.name
    if isinstance(a, float):
        if math.isnan(a):
            return "NaN"
        if math.isinf(a):
            return "Infinity" if a > 0 else "-Infinity"
        return format_double(a)
    return conv_string(a)


def _fmt_verb(verb, prec, a):
    if verb == "s":
        return _fmt_s(a)
    if verb == "d":
        if isinstance(a, float) and (math.isnan(a) or math.isinf(a)):
            return _fmt_s(a)
        _need(isinstance(a, int) and not isinstance(a, bool), "format %d", a)
        return str(int(a))
    if verb == "f":
        _need(is_num(a), "format %f", a)
        a = float(a)
        if math.isnan(a) or math.isinf(a):
            return _fmt_s(a)
        return f"{a:.{6 if prec is None else prec}f}"
    if verb == "e":
        _need(is_num(a), "format %e", a)
        a = float(a)
        if math.isnan(a) or math.isinf(a):
            return _fmt_s(a)
        return f"{a:.{6 if prec is None else prec}e}"
    if verb == "b":
        if isinstance(a, bool):
            return "1" if a else "0"
        _need(isinstance(a, int), "format %b", a)
        return format(int(a), "b")
    if verb in "xX":
        if isinstance(a, str):
            h = a.encode("utf-8").hex()
        elif isinstance(a, bytes):
            h = a.hex()
        elif isinstance(a, int) and not isinstance(a, bool):
            h = format(int(a), "x")
        else:
            raise no_overload("format %x", a)
        return h.upper() if verb == "X" else h
    if verb == "o":
        _need(isinstance(a, int) and not isinstance(a, bool), "format %o", a)
        return format(int(a), "o")
    raise CelError(f"unrecognized formatting clause {verb!r}")


# ----------------------------------------------------------------------------- Cerbos lib set helpers

_HASHABLE = (str, float, Duration, Timestamp)


def _hashable(v):
    return (isinstance(v, _HASHABLE) or (isinstance(v, int) and not isinstance(v, bool)))


def _hkey(v):
    if isinstance(v, UInt):
        return ("uint", int(v))
    if isinstance(v, float):
        return ("double", v if v != 0 else 0.0)
    if isinstance(v, int):
        return ("int", v)
    if isinstance(v, str):
        return ("string", v)
    if isinstance(v, Duration):
        return ("dur", v.ns)
    return ("ts", v.ns)


def _convert_to_set(b: list):
    """cerbos_lib.go:370-389 convertToMap: Go map keyed by ref.Val when rhs has > 3
    hashable elements -- key identity is (dynamic type, value), i.e. NO cross-type
    numeric equality, unlike the linear `find` path which uses Equal."""
    if len(b) == 0 or not _hashable(b[0]) or len(b) <= 3:
        return None
    s = set()
    for item in b:
        if not _hashable(item):
            return None
        if isinstance(item, float) and math.isnan(item):
            continue  # NaN never equals itself as a Go map key
        s.add(_hkey(item))
    return s


def _member(m, b, va):
    if m is not None:
        if not _hashable(va) and not isinstance(va, (bool, type(None), bytes, list, CelMap)):
            return False
        try:
            return _hkey(va) in m if _hashable(va) else False
        except TypeError:
            return False
    return any(cel_equal(va, x) for x in b)


def _lists(fn, a, b):
    if not isinstance(a, list) or not isinstance(b, list):
        raise no_overload(fn, a, b)


def lib_except(a, b):
    _lists("except", a, b)
    m = _convert_to_set(b)
    return [x for x in a if not _member(m, b, x)]


def lib_is_subset(a, b):
    _lists("isSubset", a, b)
    m = _convert_to_set(b)
    return all(_member(m, b, x) for x in a)


def lib_has_intersection(a, b):
    _lists("hasIntersection", a, b)
    if len(a) > len(b):
        a, b = b, a
    m = _convert_to_set(b)
    return any(_member(m, b, x) for x in a)


def lib_intersect(a, b):
    _lists("intersect", a, b)
    if len(a) > len(b):
        a, b = b, a
    m = _convert_to_set(b)
    return [x for x in a if _member(m, b, x)]


def _parse_ip(s: str):
    """Go net.ParseIP: dotted IPv4 (no leading zeros... Go >=1.17 rejects them) or IPv6 (incl. v4-mapped)."""
    try:
        if "." in s and ":" not in s:
            parts = s.split(".")
            if len(parts) != 4:
                return None
            for p in parts:
                if not p.isdigit() or len(p) > 3 or (len(p) > 1 and p[0] == "0") or int(p) > 255:
                    return None
            return ipaddress.IPv4Address(s)
        if "%" in s:
            return None
        return ipaddress.IPv6Address(s)
    except ValueError:
        return None


def lib_in_ip_range(ip_s, cidr_s):
    if not isinstance(ip_s, str) or not isinstance(cidr_s, str):
        raise no_overload("inIPAddrRange", ip_s, cidr_s)
    ip = _parse_ip(ip_s)
    if ip is None:
        raise CelError(f"invalid IP address: {ip_s}")
    if "/" not in cidr_s:
        raise CelError(f"invalid CIDR address: {cidr_s}")
    addr_s, _, bits_s = cidr_s.partition("/")
    base = _parse_ip(addr_s)
    if base is None or not bits_s.isdigit() or (len(bits_s) > 1 and bits_s[0] == "0"):
        raise CelError(f"invalid CIDR address: {cidr_s}")
    bits = int(bits_s)
    width = 32 if isinstance(base, ipaddress.IPv4Address) else 128
    if bits > width:
        raise CelError(f"invalid CIDR address: {cidr_s}")

    def to4(a):
        if isinstance(a, ipaddress.IPv6Address) and a.ipv4_mapped is not None:
            return a.ipv4_mapped
        return a
    # Go: IPNet.Contains converts both to 4-byte form when possible and requires equal length
    ip4, base4 = to4(ip), base
    if isinstance(base, ipaddress.IPv6Address):
        ip_cmp = ip if isinstance(ip, ipaddress.IPv6Address) else None
        if ip_cmp is None:
            # v4 address against v6 network: Go compares 4-byte ip with 16-byte net -> length mismatch unless
            # the network itself is a v4-mapped one (To4 succeeds)
            if base.ipv4_mapped is not None and bits >= 96:
                base4 = base.ipv4_mapped
                bits -= 96
                width = 32
                ip_cmp = ip
            else:
                return False
        else:
            if ip.ipv4_mapped is not None:
                # ip.To4() succeeds -> 4 bytes vs 16-byte net
                if base.ipv4_mapped is not None and bits >= 96:
                    base4 = base.ipv4_mapped
                    bits -= 96
                    width = 32
                    ip_cmp = ip.ipv4_mapped
                else:
                    return False
        ip4 = ip_cmp
    else:
        if not isinstance(ip4, ipaddress.IPv4Address):
            return False
    mask = ((1 << width) - 1) ^ ((1 << (width - bits)) - 1) if bits < width else (1 << width) - 1
    if bits == 0:
        mask = 0
    return (int(ip4) & mask) == (int(base4) & mask)


# ----------------------------------------------------------------------------- evaluator

_TYPE_IDENTS = {"int": "int", "uint": "uint", "double": "double", "bool": "bool", "string": "string",
                "bytes": "bytes", "list": "list", "map": "map", "null_type": "null_type", "type": "type",
                "dyn": "dyn"}


class _FailedBinding:
    __slots__ = ("err",)

    def __init__(self, err):
        self.err = err


class Evaluator:
    """Evaluates AST nodes against an activation (dict of top-level identifiers).

    Activation keys follow buildEvalVars (internal/ruletable/ruletable.go:1303-1317):
    request, R, P, runtime, constants/C, variables/V, globals/G; ``now`` is the
    batch-constant Timestamp read by now()/timeSince() (cerbos_lib.go:185-233).
    """

    def __init__(self, activation: dict, now: Timestamp | None = None):
        self.act = activation
        self.now = now

    # -- dispatch
    def eval(self, n, env=None):
        if isinstance(n, Const):
            return n.value
        if isinstance(n, Ident):
            return self._ident(n.name, env)
        if isinstance(n, Select):
            return self._select(n, env)
        if isinstance(n, Call):
            return self._call(n, env)
        if isinstance(n, ListLit):
            return [self.eval(e, env) for e in n.elems]
        if isinstance(n, MapLit):
            m = CelMap()
            for k, v in n.entries:
                kv = self.eval(k, env)
                if not (isinstance(kv, (bool, str)) or is_num(kv)):
                    raise CelError("unsupported key type")
                found, _ = m.find(kv)
                if found:
                    raise CelError("Failed with repeated key")
                m.put(kv, self.eval(v, env))
            return m
        if isinstance(n, Macro):
            return self._macro(n, env)
        raise TypeError(f"unknown node {n!r}")

    def _ident(self, name, env):
        if env is not None and isinstance(env.get(name), _FailedBinding):
            raise env[name].err
        if env is not None and name in env:
            return env[name]
        if name in self.act:
            v = self.act[name]
            if callable(v):
                v = v()
            return v
        if name in _TYPE_IDENTS:
            return CelType(_TYPE_IDENTS[name])
        raise CelError(f"undeclared reference to '{name}'")

    def _select(self, n: Select, env):
        obj = self.eval(n.operand, env)
        if n.test_only:
            if isinstance(obj, CelMap):
                found, _ = obj.find(n.field)
                return found
            if isinstance(obj, Msg):
                return obj.has(n.field)
            raise CelError(f"has() on unsupported type {type_name(obj)}")
        if isinstance(obj, CelMap):
            found, v = obj.find(n.field)
            if not found:
                raise CelError(f"no such key: {n.field}")
            return v
        if isinstance(obj, Msg):
            return obj.get(n.field)
        raise CelError(f"type '{type_name(obj)}' does not support field selection")

    def _call(self, n: Call, env):
        fn = n.fn
        if fn == "_&&_":
            return self._logic(n, env, False)
        if fn == "_||_":
            return self._logic(n, env, True)
        if fn == "_?_:_":
            c = self.eval(n.args[0], env)
            if not isinstance(c, bool):
                raise no_overload("_?_:_", c)
            return self.eval(n.args[1] if c else n.args[2], env)
        args = []
        if n.target is not None:
            args.append(self.eval(n.target, env))
        for a in n.args:
            args.append(self.eval(a, env))
        f = _FUNCS.get(fn)
        if f is None:
            raise CelError(f"unknown function {fn}")
        return f(self, args)

    def _logic(self, n, env, is_or):
        vals = []
        err = None
        for a in n.args:
            try:
                v = self.eval(a, env)
            except CelError as e:
                if err is None:
                    err = e
                continue
            if isinstance(v, bool):
                if v == is_or:
                    return is_or
                vals.append(v)
            elif err is None:
                err = no_overload(n.fn, v)
        if err is not None:
            raise err
        return not is_or

    # -- macros
    def _iter_range(self, rng, two_var):
        """Yields (k, v) pairs: list -> (index, elem); map -> (key, value)."""
        if isinstance(rng, list):
            return [(i, x) for i, x in enumerate(rng)]
        if isinstance(rng, CelMap):
            return list(rng.items())
        raise CelError(f"expression of type '{type_name(rng)}' cannot be range of a comprehension")

    def _macro(self, n: Macro, env):
        name = n.name
        env = dict(env) if env else {}
        if name == "bind":
            # cel.bind is a comprehension whose accumulator starts as `init` (ext/bindings.go): an init that fails is an error
            # VALUE held by the variable -- it surfaces only if the body reads the variable
            try:
                env[n.vars[0]] = self.eval(n.target, env)
            except CelError as e:
                env[n.vars[0]] = _FailedBinding(e)
            return self.eval(n.args[0], env)
        rng = self.eval(n.target, env)
        two = len(n.vars) == 2
        pairs = self._iter_range(rng, two)

        def bind(k, v):
            if two:
                env[n.vars[0]] = k
                env[n.vars[1]] = v
            else:
                # one-variable form iterates list elements / map keys
                env[n.vars[0]] = v if isinstance(rng, list) else k

        if name in ("all", "all2", "exists", "exists2"):
            want = name.startswith("exists")
            err = None
            for k, v in pairs:
                bind(k, v)
                try:
                    r = self.eval(n.args[0], env)
                except CelError as e:
                    err = err or e
                    continue
                if not isinstance(r, bool):
                    err = err or no_overload(name, r)
                    continue
                if r == want:
                    return want
            if err is not None:
                raise err
            return not want
        if name in ("exists_one", "exists_one2"):
            cnt = 0
            for k, v in pairs:
                bind(k, v)
                r = self.eval(n.args[0], env)
                if not isinstance(r, bool):
                    raise no_overload(name, r)
                if r:
                    cnt += 1
            return cnt == 1
        if name == "filter":
            out = []
            for k, v in pairs:
                bind(k, v)
                r = self.eval(n.args[0], env)
                if not isinstance(r, bool):
                    raise no_overload(name, r)
                if r:
                    out.append(env[n.vars[0]])
            return out
        if name == "map":
            out = []
            for k, v in pairs:
                bind(k, v)
                if len(n.args) == 2:
                    r = self.eval(n.args[0], env)
                    if not isinstance(r, bool):
                        raise no_overload(name, r)
                    if not r:
                        continue
                out.append(self.eval(n.args[-1], env))
            return out
        if name == "transformList":
            out = []
            for k, v in pairs:
                bind(k, v)
                if len(n.args) == 2:
                    r = self.eval(n.args[0], env)
                    if not isinstance(r, bool):
                        raise no_overload(name, r)
                    if not r:
                        continue
                out.append(self.eval(n.args[-1], env))
            return out
        if name == "transformMap":
            m = CelMap()
            for k, v in pairs:
                bind(k, v)
                if len(n.args) == 2:
                    r = self.eval(n.args[0], env)
                    if not isinstance(r, bool):
                        raise no_overload(name, r)
                    if not r:
                        continue
                m.put(k, self.eval(n.args[-1], env))
            return m
        if name == "transformMapEntry":
            m = CelMap()
            for k, v in pairs:
                bind(k, v)
                if len(n.args) == 2:
                    r = self.eval(n.args[0], env)
                    if not isinstance(r, bool):
                        raise no_overload(name, r)
                    if not r:
                        continue
                e = self.eval(n.args[-1], env)
                if not isinstance(e, CelMap):
                    raise no_overload(name, e)
                for ek, ev in e.items():
                    found, _ = m.find(ek)
                    if found:
                        raise CelError("insert failed: key already exists")
                    m.put(ek, ev)
            return m
        if name == "sortBy":
            if not isinstance(rng, list):
                raise no_overload("sortBy", rng)
            keys = []
            for k, v in pairs:
                bind(k, v)
                keys.append(self.eval(n.args[0], env))
            order = _sort_indices(keys)
            return [rng[i] for i in order]
        raise CelError(f"unknown macro {name}")


def _sort_indices(keys):
    if not keys:
        return []
    k0 = keys[0]
    for k in keys:
        if type_name(k) != type_name(k0) and not (is_num(k) and is_num(k0) and type_name(k) == type_name(k0)):
            raise CelError("list elements must have the same type")
    if not (is_num(k0) or isinstance(k0, (bool, str, bytes, Timestamp, Duration))):
        raise CelError("list elements must be comparable")
    import functools
    return sorted(range(len(keys)), key=functools.cmp_to_key(lambda i, j: cel_compare(keys[i], keys[j], "sort")))


# ----------------------------------------------------------------------------- function table

def _f_eq(ev, a):
    return cel_equal(a[0], a[1])


def _f_ne(ev, a):
    return not cel_equal(a[0], a[1])


def _rel(op, pred):
    def f(ev, a):
        return pred(cel_compare(a[0], a[1], op))
    return f


def _f_not(ev, a):
    if not isinstance(a[0], bool):
        raise no_overload("!_", a[0])
    return not a[0]


def _f_in(ev, a):
    x, c = a
    if isinstance(c, list):
        return any(cel_equal(x, y) for y in c)
    if isinstance(c, CelMap):
        found, _ = c.find(x)
        return found
    raise no_overload("@in", x, c)


def _index_or_error(i):
    if _is_int(i) or isinstance(i, UInt):
        return int(i)
    if isinstance(i, float) and math.isfinite(i) and i == math.floor(i):      # (a NaN or infinite index is no index)
        return int(i)
    raise CelError(f"unsupported index type '{type_name(i)}' in list")


def _f_index(ev, a):
    c, i = a
    if isinstance(c, list):
        idx = _index_or_error(i)
        if idx < 0 or idx >= len(c):
            raise CelError(f"index out of bounds: {idx}")
        return c[idx]
    if isinstance(c, CelMap):
        found, v = c.find(i)
        if not found:
            raise CelError(f"no such key: {i!r}")
        return v
    if isinstance(c, Hierarchy):
        if not _is_int(i):
            raise CelError("unsupported index type")
        if i < 0 or i >= len(c.parts):
            raise CelError("index out of range")
        return c.parts[i]
    raise no_overload("_[_]", c, i)


def _f_size(ev, a):
    v = a[0]
    if isinstance(v, (str, bytes, list, CelMap)):
        return len(v)
    if isinstance(v, Hierarchy):
        return len(v.parts)
    raise no_overload("size", v)


def _str2(fn, op):
    def f(ev, a):
        if len(a) != 2 or not isinstance(a[0], str) or not isinstance(a[1], str):
            raise no_overload(fn, *a)
        return op(a[0], a[1])
    return f


def _f_matches(ev, a):
    if len(a) != 2 or not isinstance(a[0], str) or not isinstance(a[1], str):
        raise no_overload("matches", *a)
    return _regex(a[1]).search(a[0]) is not None


def _f_char_at(ev, a):
    s, i = a
    _need(isinstance(s, str) and _is_int(i), "charAt", *a)
    if i < 0 or i > len(s):
        raise CelError(f"index out of range: {i}")
    return s[i] if i < len(s) else ""


def _f_index_of(ev, a):
    s, sub = a[0], a[1]
    _need(isinstance(s, str) and isinstance(sub, str), "indexOf", *a)
    off = 0
    if len(a) == 3:
        off = a[2]
        _need(_is_int(off), "indexOf", *a)
        if off < 0 or off > len(s):
            raise CelError(f"index out of range: {off}")
    if sub == "":
        return off
    return s.find(sub, off)


def _f_last_index_of(ev, a):
    s, sub = a[0], a[1]
    _need(isinstance(s, str) and isinstance(sub, str), "lastIndexOf", *a)
    off = len(s)
    if len(a) == 3:
        off = a[2]
        _need(_is_int(off), "lastIndexOf", *a)
        if off < 0 or off > len(s):
            raise CelError(f"index out of range: {off}")
    if sub == "":
        return off
    if off < len(sub):
        off = len(sub) - 1 if False else off
    # search for last occurrence starting at or before `off`
    return s.rfind(sub, 0, min(len(s), off + len(sub)))


def _ascii_map(lower):
    def f(ev, a):
        s = a[0]
        _need(isinstance(s, str), "lowerAscii" if lower else "upperAscii", *a)
        if lower:
            return "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in s)
        return "".join(chr(ord(c) - 32) if "a" <= c <= "z" else c for c in s)
    return f


def _f_replace(ev, a):
    _need(len(a) in (3, 4) and all(isinstance(x, str) for x in a[:3]), "replace", *a)
    s, old, new = a[:3]
    if len(a) == 4:
        _need(_is_int(a[3]), "replace", *a)
        n = a[3]
        if n < 0:
            return s.replace(old, new)
        if old == "":
            # Go strings.Replace with empty old inserts at up to n rune boundaries
            out = []
            cnt = 0
            for i, ch in enumerate(s):
                if cnt < n:
                    out.append(new)
                    cnt += 1
                out.append(ch)
            if cnt < n:
                out.append(new)
            return "".join(out)
        return s.replace(old, new, n)
    return s.replace(old, new)


def _go_split(s, sep, n):
    if n == 0:
        return []
    if sep == "":
        chars = list(s)
        if n < 0 or n >= len(chars):
            return chars
        return chars[:n - 1] + ["".join(chars[n - 1:])]
    if n < 0:
        return s.split(sep)
    return s.split(sep, n - 1)


def _f_split(ev, a):
    _need(len(a) in (2, 3) and isinstance(a[0], str) and isinstance(a[1], str), "split", *a)
    n = -1
    if len(a) == 3:
        _need(_is_int(a[2]), "split", *a)
        n = a[2]
    return _go_split(a[0], a[1], n)


def _f_join(ev, a):
    _need(len(a) in (1, 2) and isinstance(a[0], list), "join", *a)
    sep = ""
    if len(a) == 2:
        _need(isinstance(a[1], str), "join", *a)
        sep = a[1]
    for x in a[0]:
        if not isinstance(x, str):
            raise no_overload("join", *a)
    return sep.join(a[0])


def _f_substring(ev, a):
    _need(len(a) in (2, 3) and isinstance(a[0], str) and all(_is_int(x) for x in a[1:]), "substring", *a)
    s = a[0]
    start = a[1]
    end = a[2] if len(a) == 3 else len(s)
    if start < 0 or start > len(s):
        raise CelError(f"index out of range: {start}")
    if end < 0 or end > len(s):
        raise CelError(f"index out of range: {end}")
    if start > end:
        raise CelError(f"invalid substring range. start: {start}, end: {end}")
    return s[start:end]


_GO_SPACE = "\t\n\v\f\r \x85\xa0                　"


def _f_trim(ev, a):
    _need(isinstance(a[0], str), "trim", *a)
    return a[0].strip(_GO_SPACE)


def _f_str_reverse(s):
    return s[::-1]


def _f_reverse(ev, a):
    v = a[0]
    if isinstance(v, str):
        return v[::-1]
    if isinstance(v, list):
        return v[::-1]
    raise no_overload("reverse", v)


def _f_quote(ev, a):
    s = a[0]
    _need(isinstance(s, str), "strings.quote", *a)
    out = ['"']
    esc = {"\a": "\\a", "\b": "\\b", "\f": "\\f", "\n": "\\n", "\r": "\\r", "\t": "\\t", "\v": "\\v",
           "\\": "\\\\", '"': '\\"'}
    for c in s:
        out.append(esc.get(c, c))
    out.append('"')
    return "".join(out)


def _f_format(ev, a):
    _need(len(a) == 2 and isinstance(a[0], str) and isinstance(a[1], list), "format", *a)
    return _str_format(a[0], a[1])


def _ts_getter(field, adjust=0):
    def f(ev, a):
        v = a[0]
        tz = a[1] if len(a) > 1 else None
        if isinstance(v, Timestamp):
            return _ts_fields(v, tz)[field] + adjust
        raise no_overload("get" + field, *a)
    return f


def _dur_or_ts(field, dur_div, dur_mod=None):
    tsf = _ts_getter(field)

    def f(ev, a):
        v = a[0]
        if isinstance(v, Duration):
            if len(a) != 1:
                raise no_overload("get" + field, *a)
            q = _go_div(v.ns, dur_div)
            return q
        return tsf(ev, a)
    return f


def _f_timestamp_ms(ev, a):
    v = a[0]
    if isinstance(v, Duration):
        return _go_div(v.ns, 1_000_000)
    if isinstance(v, Timestamp):
        return _ts_fields(v, a[1] if len(a) > 1 else None)["ms"]
    raise no_overload("getMilliseconds", *a)


def _f_now(ev, a):
    if ev.now is None:
        raise CelError("now() called but _cerbos_now_fn not found in activation")
    return ev.now


def _f_time_since(ev, a):
    if ev.now is None:
        raise CelError("timeSince() called but _cerbos_now_fn not found in activation")
    if len(a) != 1 or not isinstance(a[0], Timestamp):
        raise no_overload("timeSince", *a)
    return Duration(ev.now.ns - a[0].ns)


def _f_hierarchy(ev, a):
    if len(a) == 1:
        v = a[0]
        if isinstance(v, Hierarchy):
            return v
        if isinstance(v, str):
            return Hierarchy(v.split("."))
        if isinstance(v, list):
            for x in v:
                if not isinstance(x, str):
                    raise CelError("failed to convert list to string slice")
            return Hierarchy(v)
        raise no_overload("hierarchy", v)
    if len(a) == 2 and isinstance(a[0], str) and isinstance(a[1], str):
        if a[1] == "":
            return Hierarchy(list(a[0]))
        return Hierarchy(a[0].split(a[1]))
    raise no_overload("hierarchy", *a)


def _hier2(fn):
    def f(ev, a):
        if len(a) != 2 or not isinstance(a[0], Hierarchy) or not isinstance(a[1], Hierarchy):
            raise no_overload(fn.__name__, *a)
        return fn(a[0].parts, a[1].parts)
    return f


def _h_ancestor_of(h, c):
    return len(c) > len(h) and c[:len(h)] == h


def _h_common(h, o):
    short, long_ = (h, o) if len(o) >= len(h) else (o, h)
    if len(long_) == len(short):
        long_ = long_[:-1]
        short = short[:-1]
    out = []
    for i, s in enumerate(short):
        if long_[i] != s:
            break
        out.append(s)
    return Hierarchy(out)


def _h_imm_parent(h, c):
    return len(c) == len(h) + 1 and c[:len(h)] == h


def _h_sibling(h, o):
    return len(o) == len(h) and h[:-1] == o[:-1]


def _h_overlaps(h, o):
    short, long_ = (h, o) if len(o) >= len(h) else (o, h)
    return long_[:len(short)] == short


def _f_type(ev, a):
    return CelType(type_name(a[0]))


def _f_lists_range(ev, a):
    _need(len(a) == 1 and _is_int(a[0]), "lists.range", *a)
    return list(range(a[0]))


def _f_distinct(ev, a):
    _need(isinstance(a[0], list), "distinct", *a)
    out = []
    for x in a[0]:
        if not any(cel_equal(x, y) for y in out):
            out.append(x)
    return out


def _flatten(lst, depth):
    out = []
    for x in lst:
        if isinstance(x, list) and depth > 0:
            out.extend(_flatten(x, depth - 1))
        else:
            out.append(x)
    return out


def _f_flatten(ev, a):
    _need(isinstance(a[0], list), "flatten", *a)
    depth = 1
    if len(a) == 2:
        _need(_is_int(a[1]), "flatten", *a)
        depth = a[1]
        if depth < 0:
            raise CelError("level must be non-negative")
    return _flatten(a[0], depth)


def _f_slice(ev, a):
    _need(len(a) == 3 and isinstance(a[0], list) and _is_int(a[1]) and _is_int(a[2]), "slice", *a)
    lst, s, e = a
    if s < 0 or e < 0:
        raise CelError(f"cannot slice({s}, {e}), negative indexes not supported")
    if s > e:
        raise CelError(f"cannot slice({s}, {e}), start index must be less than or equal to end index")
    if e > len(lst):
        raise CelError(f"cannot slice({s}, {e}), list is length {len(lst)}")
    return lst[s:e]


def _f_sort(ev, a):
    _need(isinstance(a[0], list), "sort", *a)
    order = _sort_indices(a[0])
    return [a[0][i] for i in order]


def _f_first(ev, a):
    _need(isinstance(a[0], list), "first", *a)
    if not a[0]:
        raise CelError("optional.none() dereference")
    return a[0][0]


def _f_last(ev, a):
    _need(isinstance(a[0], list), "last", *a)
    if not a[0]:
        raise CelError("optional.none() dereference")
    return a[0][-1]


def _minmax(name, pick_greater):
    def f(ev, a):
        vals = a
        if len(a) == 1:
            if isinstance(a[0], list):
                vals = a[0]
                if not vals:
                    raise CelError(f"math.@{name}(list) argument must not be empty")
            elif is_num(a[0]):
                return a[0]
            else:
                raise no_overload(name, *a)
        best = None
        for v in vals:
            if not is_num(v):
                raise no_overload(name, *a)
            if best is None:
                best = v
                continue
            c = num_compare(v, best, for_equality=True)
            if c is None:
                # NaN handling: cel-go uses Compare which errors... keep first
                raise CelError("NaN values cannot be ordered")
            if (c > 0) == pick_greater and c != 0:
                best = v
        return best
    return f


def _math1(name, fi=None, fu=None, fd=None):
    def f(ev, a):
        v = a[0]
        if len(a) != 1:
            raise no_overload(name, *a)
        if isinstance(v, UInt) and fu:
            return fu(v)
        if _is_int(v) and fi:
            return fi(v)
        if isinstance(v, float) and fd:
            return fd(v)
        raise no_overload(name, v)
    return f


def _round_half_away(d):
    """Go's math.Round (exact: |d| - floor(|d|) is computed without rounding error, unlike floor(|d| + 0.5))"""
    if math.isnan(d) or math.isinf(d):
        return d
    f = math.floor(abs(d))
    return math.copysign(f + 1.0 if abs(d) - f >= 0.5 else f, d)


def _keep_zero_sign(fn, d):
    """Go's math.Ceil / Floor / Trunc: +-Inf and NaN unchanged, a zero result keeps the argument's sign (Ceil(-0.5) = -0)"""
    if math.isnan(d) or math.isinf(d):
        return d
    return math.copysign(0.0, d) if fn(d) == 0 else float(fn(d))


def _abs_int(v):
    if v == INT64_MIN:
        raise CelError("integer overflow")
    return abs(v)


def _sign_d(d):
    if math.isnan(d):
        return d
    return 0.0 if d == 0 else math.copysign(1.0, d)


def _bit2(name, op):
    def f(ev, a):
        x, y = a
        if _is_int(x) and _is_int(y):
            r = op(x & UINT64_MAX, y & UINT64_MAX) & UINT64_MAX
            return r - (1 << 64) if r > INT64_MAX else r
        if isinstance(x, UInt) and isinstance(y, UInt):
            return UInt(op(int(x), int(y)) & UINT64_MAX)
        raise no_overload(name, x, y)
    return f


def _f_bit_not(ev, a):
    x = a[0]
    if _is_int(x):
        return ~x
    if isinstance(x, UInt):
        return UInt(~int(x) & UINT64_MAX)
    raise no_overload("math.bitNot", x)


def _shift(left):
    def f(ev, a):
        x, n = a
        if not _is_int(n):
            raise no_overload("math.bitShift", x, n)
        if n < 0:
            raise CelError("math.bitShift() negative offset")
        if _is_int(x):
            if n >= 64:
                return 0
            u = x & UINT64_MAX
            r = (u << n) & UINT64_MAX if left else u >> n
            return r - (1 << 64) if r > INT64_MAX else r
        if isinstance(x, UInt):
            if n >= 64:
                return UInt(0)
            return UInt((int(x) << n) & UINT64_MAX if left else int(x) >> n)
        raise no_overload("math.bitShift", x, n)
    return f


def _f_b64enc(ev, a):
    _need(isinstance(a[0], bytes), "base64.encode", *a)
    return _b64.b64encode(a[0]).decode("ascii")


_B64_ALPHABET = frozenset("ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/")


def _f_b64dec(ev, a):
    """cel-go ext.Encoders: base64.StdEncoding.DecodeString, then RawStdEncoding.  Go's decoder (encoding/base64) skips CR / LF
    anywhere; padded text has a length that is a multiple of four with one or two '=' at the very end and nowhere else;
    unpadded text may end in a quantum of two or three characters; not being Strict(), non-zero trailing bits are dropped.
    (Python's decoder is more forgiving about misplaced padding, so the shape is checked here.)"""
    _need(isinstance(a[0], str), "base64.decode", *a)
    s = a[0].replace("\r", "").replace("\n", "")
    body = s.rstrip("=")
    pad = len(s) - len(body)
    if pad:
        if pad > 2 or len(s) % 4 != 0:
            raise CelError("illegal base64 data")
    elif len(s) % 4 == 1:
        raise CelError("illegal base64 data")
    if not all(c in _B64_ALPHABET for c in body):
        raise CelError("illegal base64 data")
    return _b64.b64decode(body + "=" * (-len(body) % 4))


def _f_sqrt(ev, a):
    v = a[0]
    if not is_num(v):
        raise no_overload("math.sqrt", v)
    v = float(v)
    return math.nan if v < 0 else math.sqrt(v)


def _conv(fn):
    def f(ev, a):
        if len(a) != 1:
            raise no_overload(fn.__name__, *a)
        return fn(a[0])
    return f


def _lib2(fn):
    def f(ev, a):
        if len(a) != 2:
            raise no_overload(fn.__name__, *a)
        return fn(a[0], a[1])
    return f


def _f_spiffe_id(ev, a):
    if len(a) == 1 and isinstance(a[0], SpiffeID):
        return a[0]
    if len(a) == 1 and isinstance(a[0], str):
        return SpiffeID(a[0])
    raise no_overload("spiffeID", *a)


def _f_spiffe_td(ev, a):
    if len(a) == 1 and isinstance(a[0], SpiffeTD):
        return a[0]
    if len(a) == 1 and isinstance(a[0], SpiffeID):
        return SpiffeTD(a[0].td)
    if len(a) == 1 and isinstance(a[0], str):
        return SpiffeTD(spiffe_parse_td(a[0]))
    raise no_overload("spiffeTrustDomain", *a)


def _f_spiffe_match_exact(ev, a):
    if len(a) == 1 and isinstance(a[0], SpiffeID):
        return SpiffeMatcher("exact", a[0].id)
    if len(a) == 1 and isinstance(a[0], str):
        return SpiffeMatcher("exact", SpiffeID(a[0]).id)
    raise no_overload("spiffeMatchExact", *a)


def _f_spiffe_match_one_of(ev, a):
    if len(a) != 1 or not isinstance(a[0], list):
        raise no_overload("spiffeMatchOneOf", *a)
    if all(isinstance(x, SpiffeID) for x in a[0]):
        return SpiffeMatcher("oneof", {x.id for x in a[0]})
    if all(isinstance(x, str) for x in a[0]):
        try:
            return SpiffeMatcher("oneof", {SpiffeID(x).id for x in a[0]})
        except CelError:
            pass
    raise no_overload("spiffeMatchOneOf", *a)


def _f_spiffe_match_td(ev, a):
    if len(a) == 1 and isinstance(a[0], SpiffeTD):
        return SpiffeMatcher("td", a[0].name)
    if len(a) == 1 and isinstance(a[0], str):
        return SpiffeMatcher("td", spiffe_parse_td(a[0]))
    raise no_overload("spiffeMatchTrustDomain", *a)


def _f_spiffe_matches_id(ev, a):
    if len(a) != 2 or not isinstance(a[0], SpiffeMatcher):
        raise no_overload("matchesID", *a)
    if isinstance(a[1], SpiffeID):
        return a[0].matches(a[1])
    if isinstance(a[1], str):
        return a[0].matches(SpiffeID(a[1]))
    raise no_overload("matchesID", *a)


def _f_spiffe_member_of(ev, a):
    if len(a) != 2 or not isinstance(a[0], SpiffeID) or not isinstance(a[1], SpiffeTD):
        raise no_overload("isMemberOf", *a)
    return a[0].td == a[1].name


def _spiffe_recv(fn, cls, f):
    def g(ev, a):
        if len(a) != 1 or not isinstance(a[0], cls):
            raise no_overload(fn, *a)
        return f(a[0])
    return g


def _f_id(ev, a):
    if len(a) == 1 and isinstance(a[0], SpiffeTD):   # spiffeTrustDomain.id(): the fully qualified trust domain id
        return "spiffe://" + a[0].name
    return a[0]                                        # cerbos_lib.go: id(x) = x


_FUNCS = {
    "_==_": _f_eq, "_!=_": _f_ne,
    "spiffeID": _f_spiffe_id, "spiffeTrustDomain": _f_spiffe_td, "spiffeMatchAny": lambda ev, a: SpiffeMatcher("any") if not a else (_ for _ in ()).throw(no_overload("spiffeMatchAny", *a)),
    "spiffeMatchExact": _f_spiffe_match_exact, "spiffeMatchOneOf": _f_spiffe_match_one_of, "spiffeMatchTrustDomain": _f_spiffe_match_td,
    "matchesID": _f_spiffe_matches_id, "isMemberOf": _f_spiffe_member_of,
    "path": _spiffe_recv("path", SpiffeID, lambda s: s.id[s.pathidx:]), "trustDomain": _spiffe_recv("trustDomain", SpiffeID, lambda s: SpiffeTD(s.td)),
    "name": _spiffe_recv("name", SpiffeTD, lambda t: t.name),
    "_<_": _rel("_<_", lambda c: c < 0), "_<=_": _rel("_<=_", lambda c: c <= 0),
    "_>_": _rel("_>_", lambda c: c > 0), "_>=_": _rel("_>=_", lambda c: c >= 0),
    "_+_": lambda ev, a: op_add(*a), "_-_": lambda ev, a: op_sub(*a), "_*_": lambda ev, a: op_mul(*a),
    "_/_": lambda ev, a: op_div(*a), "_%_": lambda ev, a: op_mod(*a), "-_": lambda ev, a: op_neg(*a),
    "!_": _f_not, "@in": _f_in, "_[_]": _f_index, "size": _f_size,
    "int": _conv(conv_int), "uint": _conv(conv_uint), "double": _conv(conv_double), "string": _conv(conv_string),
    "bool": _conv(conv_bool), "bytes": _conv(conv_bytes), "timestamp": _conv(conv_timestamp),
    "duration": _conv(conv_duration), "dyn": lambda ev, a: a[0], "type": _f_type, "id": _f_id,
    "contains": _str2("contains", lambda s, t: t in s), "startsWith": _str2("startsWith", lambda s, t: s.startswith(t)),
    "endsWith": _str2("endsWith", lambda s, t: s.endswith(t)), "matches": _f_matches,
    "charAt": _f_char_at, "indexOf": _f_index_of, "lastIndexOf": _f_last_index_of,
    "lowerAscii": _ascii_map(True), "upperAscii": _ascii_map(False), "replace": _f_replace, "split": _f_split,
    "join": _f_join, "substring": _f_substring, "trim": _f_trim, "reverse": _f_reverse, "format": _f_format,
    "strings.quote": _f_quote,
    "getFullYear": _ts_getter("year"), "getMonth": _ts_getter("month", -1), "getDayOfYear": _ts_getter("doy"),
    "getDayOfMonth": _ts_getter("day", -1), "getDate": _ts_getter("day"), "getDayOfWeek": _ts_getter("dow"),
    "getHours": _dur_or_ts("hour", 3_600_000_000_000), "getMinutes": _dur_or_ts("minute", 60_000_000_000),
    "getSeconds": _dur_or_ts("second", 1_000_000_000), "getMilliseconds": _f_timestamp_ms,
    "now": _f_now, "timeSince": _f_time_since,
    "except": _lib2(lib_except), "intersect": _lib2(lib_intersect),
    "hasIntersection": _lib2(lib_has_intersection), "has_intersection": _lib2(lib_has_intersection),
    "isSubset": _lib2(lib_is_subset), "is_subset": _lib2(lib_is_subset),
    "inIPAddrRange": _lib2(lib_in_ip_range),
    "hierarchy": _f_hierarchy,
    "ancestorOf": _hier2(_h_ancestor_of), "commonAncestors": _hier2(_h_common),
    "descendentOf": _hier2(lambda h, p: _h_ancestor_of(p, h)),
    "immediateChildOf": _hier2(lambda h, p: _h_imm_parent(p, h)), "immediateParentOf": _hier2(_h_imm_parent),
    "overlaps": _hier2(_h_overlaps), "siblingOf": _hier2(_h_sibling),
    "lists.range": _f_lists_range, "distinct": _f_distinct, "flatten": _f_flatten, "slice": _f_slice,
    "sort": _f_sort, "first": _f_first, "last": _f_last,
    "math.greatest": _minmax("max", True), "math.least": _minmax("min", False),
    "math.ceil": _math1("math.ceil", fd=lambda d: _keep_zero_sign(math.ceil, d)),
    "math.floor": _math1("math.floor", fd=lambda d: _keep_zero_sign(math.floor, d)),
    "math.round": _math1("math.round", fd=_round_half_away),
    "math.trunc": _math1("math.trunc", fd=lambda d: _keep_zero_sign(math.trunc, d)),
    "math.abs": _math1("math.abs", fi=_abs_int, fu=lambda u: u, fd=abs),
    "math.sign": _math1("math.sign", fi=lambda i: (i > 0) - (i < 0), fu=lambda u: UInt(1 if u > 0 else 0), fd=_sign_d),
    "math.isNaN": _math1("math.isNaN", fd=math.isnan), "math.isInf": _math1("math.isInf", fd=math.isinf),
    "math.isFinite": _math1("math.isFinite", fd=math.isfinite),
    "math.bitAnd": _bit2("math.bitAnd", lambda x, y: x & y), "math.bitOr": _bit2("math.bitOr", lambda x, y: x | y),
    "math.bitXor": _bit2("math.bitXor", lambda x, y: x ^ y), "math.bitNot": _f_bit_not,
    "math.bitShiftLeft": _shift(True), "math.bitShiftRight": _shift(False), "math.sqrt": _f_sqrt,
    "base64.encode": _f_b64enc, "base64.decode": _f_b64dec,
}


def eval_expr(node, activation: dict, now: Timestamp | None = None):
    """Evaluate; raises CelError for CEL error values."""
    return Evaluator(activation, now).eval(node)
