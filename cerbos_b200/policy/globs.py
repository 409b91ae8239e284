"""Glob matching for actions / resources / roles (host side).

Restates internal/util/globs_common.go:11-87 (``glob.Compile(expr, ':')`` with the
lone ``*`` -> ``**`` fix-up at :74-81) over the published syntax of
github.com/gobwas/glob v0.2.3 (go.mod:42; source outside the reference tree):
``*`` = any run of non-separator chars, ``**`` = any run, ``?`` = one non-separator
char, ``[abc]``/``[a-z]``/``[!abc]`` classes, ``{a,b}`` alternatives, ``\\`` escape.

A rule-table key is treated as a glob iff it contains ``*``
(internal/ruletable/internal/glob_map.go:60-75); everything else is a literal.
Parity note: only ``*``, ``**`` and ``prefix:*`` forms are pinned by reference
goldens; classes/alternatives follow the library's documentation ("parity unpinned").
"""
from __future__ import annotations

import functools
import re

SEP = ":"


def is_glob(key: str) -> bool:
    return "*" in key


def _translate(p: str, i: int, in_alt: bool):
    out = []
    n = len(p)
    while i < n:
        c = p[i]
        if c == "\\":
            i += 1
            if i >= n:
                raise ValueError("dangling escape in glob")
            out.append(re.escape(p[i]))
            i += 1
        elif c == "*":
            j = i
            while j < n and p[j] == "*":
                j += 1
            out.append(".*" if j - i >= 2 else f"[^{re.escape(SEP)}]*")
            i = j
        elif c == "?":
            out.append(f"[^{re.escape(SEP)}]")
            i += 1
        elif c == "[":
            j = i + 1
            neg = j < n and p[j] == "!"
            if neg:
                j += 1
            k = j
            body = []
            while k < n and p[k] != "]":
                if p[k] == "\\" and k + 1 < n:
                    body.append(re.escape(p[k + 1]))
                    k += 2
                elif p[k] == "-" and body and k + 1 < n and p[k + 1] != "]":
                    body.append("-")
                    k += 1
                else:
                    body.append(re.escape(p[k]))
                    k += 1
            if k >= n:
                raise ValueError("unterminated character class in glob")
            out.append("[" + ("^" if neg else "") + "".join(body) + "]")
            i = k + 1
        elif c == "{":
            alts = []
            i += 1
            while True:
                sub, i, term = _translate(p, i, True)
                alts.append(sub)
                if term == "}":
                    break
                if term is None:
                    raise ValueError("unterminated alternatives in glob")
            out.append("(?:" + "|".join(alts) + ")")
        elif in_alt and c == ",":
            return "".join(out), i + 1, ","
        elif in_alt and c == "}":
            return "".join(out), i + 1, "}"
        else:
            out.append(re.escape(c))
            i += 1
    return "".join(out), i, None


@functools.lru_cache(maxsize=4096)
def _compile(glob_expr: str):
    if glob_expr == "*":
        glob_expr = "**"
    try:
        rx, _, _ = _translate(glob_expr, 0, False)
        return re.compile(rx, re.DOTALL)
    except (ValueError, re.error):
        return None


def matches_glob(glob_expr: str, val: str) -> bool:
    """util.MatchesGlob: invalid patterns match nothing."""
    g = _compile(glob_expr)
    return g is not None and g.fullmatch(val) is not None


def key_matches(key: str, val: str) -> bool:
    """GlobMap semantics: literal equality, or glob match when the key contains '*'."""
    if key == val:
        return True
    return is_glob(key) and matches_glob(key, val)
