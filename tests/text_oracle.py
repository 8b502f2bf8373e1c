"""Python restatement of the device text parser's grammar and exact conversion (csrc/textparse.cu, pn2_api.h
PN2_TEXT_*): the verdict for every file, and the float32 value of every field the device converts."""
from __future__ import annotations

import numpy as np

OK, SYNTAX, FIELDS, BLANK, CR, COMMENT, INEXACT = range(7)
WHITESPACE, COMMA = 0, 1
_EXP_CAP = 1 << 20
_POW10 = [float(10 ** k) for k in range(23)]


def _reason(c: str) -> int:
    return CR if c == "\r" else COMMENT if c == "#" else SYNTAX


def parse_field(s: str, p: int):
    """(status, value, p past the field) of the field at s[p:]."""
    at = lambda q: s[q] if q < len(s) else ""  # noqa: E731
    neg = False
    c = at(p)
    if c and c in "+-":
        neg, p = c == "-", p + 1
        c = at(p)
    m = nd = frac = digits = 0
    while c and c in "0123456789":
        if not (m == 0 and c == "0"):
            if nd < 17:
                m = m * 10 + int(c)
            nd += 1
        digits += 1
        p += 1
        c = at(p)
    if c == ".":
        p += 1
        c = at(p)
        if not (c and c in "0123456789"):
            return _reason(c), None, p
        while c and c in "0123456789":
            frac = min(frac + 1, _EXP_CAP)
            if not (m == 0 and c == "0"):
                if nd < 17:
                    m = m * 10 + int(c)
                nd += 1
            digits += 1
            p += 1
            c = at(p)
    if not digits:
        return _reason(c), None, p
    e = 0
    if c and c in "eE":
        p += 1
        c = at(p)
        eneg = False
        if c and c in "+-":
            eneg, p = c == "-", p + 1
            c = at(p)
        if not (c and c in "0123456789"):
            return _reason(c), None, p
        while c and c in "0123456789":
            e = min(e * 10 + int(c), _EXP_CAP)
            p += 1
            c = at(p)
        if eneg:
            e = -e
    e -= frac
    if nd > 16 or m > 2 ** 53 or not -22 <= e <= 22:
        return INEXACT, None, p
    d = float(m)
    if e > 0:
        d = d * _POW10[e]
    elif e < 0:
        d = d / _POW10[-e]
    return OK, np.float32(-d if neg else d), p


def parse_line(s: str, ncol: int, delim: int):
    """(status, values) of one line without its terminator (a "\\r" before "\\n" already removed)."""
    p, vals = 0, []
    if delim == WHITESPACE:
        while p < len(s) and s[p] in " \t":
            p += 1
    if p == len(s):
        return BLANK, None
    f = 0
    while True:
        if f == ncol:
            return FIELDS, None
        r, v, p = parse_field(s, p)
        if r != OK:
            return r, None
        vals.append(v)
        if p == len(s):
            return (OK, vals) if f + 1 == ncol else (FIELDS, None)
        c = s[p]
        if delim == COMMA:
            if c != ",":
                return _reason(c), None
            p += 1
        else:
            if c not in " \t":
                return _reason(c), None
            while p < len(s) and s[p] in " \t":
                p += 1
            if p == len(s):
                return (OK, vals) if f + 1 == ncol else (FIELDS, None)
        f += 1


def classify_file(data: bytes, ncol: int, delim: int):
    """(status, rows): the device's verdict on one file and, when it is OK, its (rows, ncol) float32 table."""
    s = data.decode("latin-1")
    lines = s.split("\n")
    terminated = [True] * (len(lines) - 1) + [False]
    if lines[-1] == "":  # the file ends with its terminator, or is empty
        lines, terminated = lines[:-1], terminated[:-1]
    out = []
    for line, term in zip(lines, terminated):
        if term and line.endswith("\r"):
            line = line[:-1]
        r, vals = parse_line(line, ncol, delim)
        if r != OK:
            return r, None
        out.append(vals)
    return OK, np.array(out, np.float32).reshape(len(out), ncol)


def convert(s: str):
    """The device's float32 of one field string, or None when it is outside the grammar or the exact path."""
    r, v, p = parse_field(s, 0)
    return v if r == OK and p == len(s) else None
