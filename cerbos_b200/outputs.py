"""Rule outputs: decoding the records of cgpu_check_outputs into the reference's OutputEntry list.

A record (layout.py: OUT_TAGS) holds CEL-typed values; the conversion to google.protobuf.Value that the reference applies
(ruletable.go:1443-1482, cel-go's ConvertToNative(*structpb.Value)) happens here:

  * an evaluation error gives an entry with no value (None);
  * numbers become doubles, bytes base64 text, timestamps RFC 3339 text in UTC, durations seconds followed by "s";
  * map keys are written in their string form;
  * a value with no Value form anywhere inside it (a type, a SPIFFE id) gives "<failed to convert evaluation to protobuf value>".
"""
from __future__ import annotations

import base64
import datetime
import math
import struct

from .table import layout as L

NOT_CONVERTIBLE = "<failed to convert evaluation to protobuf value>"
_T = L.OUT_TAGS


class _NoForm(Exception):
    pass


def _double_text(d: float) -> str:
    """strconv.FormatFloat(d, 'f', -1, 64): the shortest digits that round-trip, never an exponent."""
    if math.isnan(d):
        return "NaN"
    if math.isinf(d):
        return "+Inf" if d > 0 else "-Inf"
    sign = "-" if math.copysign(1, d) < 0 else ""
    mant, _, exp = repr(abs(d)).partition("e")
    ip, _, fp = mant.partition(".")
    digits, point = ip + fp, len(ip) + (int(exp) if exp else 0)
    if point <= 0:
        digits, point = "0" * (1 - point) + digits, 1
    digits += "0" * max(0, point - len(digits))
    whole, frac = digits[:point].lstrip("0") or "0", digits[point:].rstrip("0")
    return sign + whole + ("." + frac if frac else "")


def _frac(ns: int) -> str:
    return "." + f"{ns:09d}".rstrip("0") if ns else ""


def timestamp_text(ns: int) -> str:
    s, sub = divmod(ns, 1_000_000_000)
    t = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=s)
    return f"{t.year:04d}-{t.month:02d}-{t.day:02d}T{t.hour:02d}:{t.minute:02d}:{t.second:02d}{_frac(sub)}Z"


def duration_text(ns: int) -> str:
    s, sub = divmod(abs(ns), 1_000_000_000)
    return f"{'-' if ns < 0 else ''}{s}{_frac(sub)}s"


class _Reader:
    def __init__(self, buf: bytes, pos: int):
        self.buf, self.pos = buf, pos

    def take(self, fmt: str):
        v = struct.unpack_from(fmt, self.buf, self.pos)
        self.pos += struct.calcsize(fmt)
        return v[0]

    def raw(self, n: int) -> bytes:
        b = bytes(self.buf[self.pos:self.pos + n])
        self.pos += n
        return b

    def value(self, key=False):
        """The next value in its protobuf Value form (key: its string form); _NoForm where it has none."""
        tag = self.take("<B")
        if tag == _T["NO_VALUE"] or tag == _T["NULL"]:
            if key:
                raise _NoForm()
            return None
        if tag == _T["BOOL"]:
            b = self.take("<B") != 0
            return ("true" if b else "false") if key else b
        if tag in (_T["INT"], _T["UINT"]):
            i = self.take("<q" if tag == _T["INT"] else "<Q")
            return str(i) if key else float(i)
        if tag == _T["DOUBLE"]:
            d = self.take("<d")
            return _double_text(d) if key else d
        if tag in (_T["STRING"], _T["BYTES"]):
            b = self.raw(self.take("<I"))
            if tag == _T["STRING"]:
                return b.decode("utf-8")
            if key:
                try:
                    return b.decode("utf-8")
                except UnicodeDecodeError:
                    raise _NoForm() from None
            return base64.b64encode(b).decode("ascii")
        if tag == _T["TIMESTAMP"]:
            return timestamp_text(self.take("<q"))
        if tag == _T["DURATION"]:
            return duration_text(self.take("<q"))
        if tag == _T["LIST"] and not key:
            n = self.take("<I")
            return [self.value() for _ in range(n)]
        if tag == _T["MAP"] and not key:
            n = self.take("<I")
            out = {}
            for _ in range(n):
                k = self.value(key=True)
                out[k] = self.value()
            return out
        raise _NoForm()

    def skip_value(self):
        tag = self.take("<B")
        if tag == _T["BOOL"]:
            self.pos += 1
        elif tag in (_T["INT"], _T["UINT"], _T["DOUBLE"], _T["TIMESTAMP"], _T["DURATION"]):
            self.pos += 8
        elif tag in (_T["STRING"], _T["BYTES"]):
            self.pos += self.take("<I")
        elif tag == _T["LIST"]:
            for _ in range(self.take("<I")):
                self.skip_value()
        elif tag == _T["MAP"]:
            for _ in range(2 * self.take("<I")):
                self.skip_value()


def decode_record(rec, sources, actions) -> list:
    """One request's record -> [{"src", "action", "val"}] in emission order.  sources: MANIFEST output_sources; actions:
    the request's actions (the entries carry action indices)."""
    r = _Reader(rec, 0)
    needed, n = r.take("<I"), r.take("<I")
    if needed > len(rec):
        raise ValueError(f"output record needs {needed} bytes, has {len(rec)}")
    out = []
    for _ in range(n):
        action, _pad, src = r.take("<H"), r.take("<H"), r.take("<I")
        start = r.pos
        try:
            val = r.value()
        except _NoForm:
            r.pos = start
            r.skip_value()
            val = NOT_CONVERTIBLE
        out.append({"src": sources[src], "action": actions[action], "val": val})
    return out


def decode(records, stride: int, manifest: dict, actions_per_request) -> list:
    """Every request's entries: records is the n_requests * stride byte buffer cgpu_check_outputs filled."""
    buf = memoryview(records).cast("B")
    sources = manifest.get("output_sources", [])
    return [decode_record(buf[i * stride:(i + 1) * stride], sources, acts) for i, acts in enumerate(actions_per_request)]
