"""CPU restatement of the string-producing functions (expressions.py Substring / Concat / ConcatWs / StringTrim* / StringLPad /
StringRPad / Length) on Python bytes, stepping code points the way UTF8String does: by the width each lead byte declares
(numBytesForFirstByte), so ill-formed bytes give the reference's answer.  None is NULL.

A truncated lead byte at the end of a value declares more bytes than remain.  The trims clamp such a character to the value, as the
reference does; substring and pad cut at the value's end there too (the reference's copy would read past the value).
"""
from __future__ import annotations

INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31


def step(b: int) -> int:
    """UTF8String.numBytesForFirstByte"""
    return 1 if b < 0xC2 else 2 if b < 0xE0 else 3 if b < 0xF0 else 4 if b < 0xF5 else 1


def num_chars(s: bytes) -> int:
    i = c = 0
    while i < len(s):
        i += step(s[i])
        c += 1
    return c


def _advance(s: bytes, i: int, c: int, upto: int):
    while i < len(s) and c < upto:
        i += step(s[i])
        c += 1
    return i, c


def substring(s: bytes, start: int, until: int) -> bytes:
    """UTF8String.substring(start, until), in code points"""
    if until <= start or start >= len(s):
        return b""
    i, c = _advance(s, 0, 0, start)
    j = i
    i = len(s) if until == INT_MAX else _advance(s, i, c, until)[0]
    return s[min(j, len(s)):min(i, len(s))]


def substring_sql(s, pos, length=INT_MAX):
    if s is None or pos is None or length is None:
        return None
    start = pos - 1 if pos > 0 else (num_chars(s) + pos if pos < 0 else 0)
    end = max(INT_MIN, min(INT_MAX, start + length))
    return substring(s, start, end)


def concat(*xs):
    return None if any(x is None for x in xs) else b"".join(xs)


def concat_ws(sep, *xs):
    return None if sep is None else sep.join(x for x in xs if x is not None)


def _chars(s: bytes, frm: int = 0):
    """(start, end) of every code point from byte frm, the last one clamped to the value"""
    i = frm
    while i < len(s):
        e = min(i + step(s[i]), len(s))
        yield i, e
        i = e


def _ltrim_at(s: bytes, trim: bytes) -> int:
    for a, e in _chars(s):
        if s[a:e] not in trim:        # UTF8String.find: the character's bytes anywhere in the set's bytes
            return a
    return len(s)


def _rtrim_end(s: bytes, trim: bytes, frm: int) -> int:
    end = frm
    for a, e in _chars(s, frm):
        if s[a:e] not in trim:
            end = e
    return end


_ABSENT = object()


def trim(s, trim_str=_ABSENT):
    if s is None or trim_str is None:
        return None
    if trim_str is _ABSENT:
        return s.strip(b" ")
    a = _ltrim_at(s, trim_str)
    return s[a:_rtrim_end(s, trim_str, a)]


def ltrim(s, trim_str=_ABSENT):
    if s is None or trim_str is None:
        return None
    if trim_str is _ABSENT:
        return s.lstrip(b" ")
    return s[_ltrim_at(s, trim_str):]


def rtrim(s, trim_str=_ABSENT):
    if s is None or trim_str is None:
        return None
    if trim_str is _ABSENT:
        return s.rstrip(b" ")
    return s[:_rtrim_end(s, trim_str, 0)]


def _pad(s, length, pad, left):
    if s is None or length is None or pad is None:
        return None
    if length <= 0:
        return b""
    spaces = length - num_chars(s)
    if spaces <= 0 or not pad:
        return substring(s, 0, length)
    pc = num_chars(pad)
    count = spaces // pc
    filler = pad * count + substring(pad, 0, spaces - pc * count)
    return filler + s if left else s + filler


def lpad(s, length, pad=b" "):
    return _pad(s, length, pad, True)


def rpad(s, length, pad=b" "):
    return _pad(s, length, pad, False)


def length(s):
    return None if s is None else num_chars(s)


def evaluate(e, row: dict):
    """The value of a spark_b200.expressions string function (or column / literal) for one row of bytes values."""
    from spark_b200 import expressions as E
    if isinstance(e, E.AttributeReference):
        return row[e.name]
    if isinstance(e, E.Literal):
        return None if e.value is None else (e.value if isinstance(e.value, bytes) else e.value.encode())
    if isinstance(e, E.Substring):
        return substring_sql(evaluate(e.child, row), e.pos, e.len)
    if isinstance(e, E.ConcatWs):
        return concat_ws(e.sep, *[evaluate(c, row) for c in e.children])
    if isinstance(e, E.Concat):
        return concat(*[evaluate(c, row) for c in e.children])
    if isinstance(e, E._Trim):
        f = {"trim": trim, "ltrim": ltrim, "rtrim": rtrim}[e.name]
        return f(evaluate(e.child, row), e.trim) if e.given else f(evaluate(e.child, row))
    if isinstance(e, E._Pad):
        return (lpad if e.name == "lpad" else rpad)(evaluate(e.child, row), e.len, e.pad)
    if isinstance(e, E.Length):
        return length(evaluate(e.child, row))
    raise TypeError(e)
