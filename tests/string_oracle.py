"""CPU restatement of the string tests (expressions.py StartsWith / EndsWith / Contains / Like / In / OctetLength and comparisons
with a string literal) on Python bytes and str, independent of the engine's matchers.

`eval_expr(e, table)` takes the sexpr() form: every string test is evaluated here into a (value, valid) column, substituted by a
reference to it, and the rest of the program goes to oracle.eval_expr.  The semantics are Spark's with the UTF8_BINARY collation:
comparisons by unsigned bytes (binary_compare), IN is TRUE on a match, else NULL when the list holds NULL, else FALSE; LIKE is
StringUtils.escapeLikeRegex run through `re` with DOTALL on the decoded string; a NULL string gives NULL."""
import re

import numpy as np
import pyarrow as pa

from oracle import oracle as O

STRING_OPS = ("str_cmp", "in", "starts_with", "ends_with", "contains", "like", "octet_length")


class LikePatternError(ValueError):
    pass


def like_regex(pattern: str, escape: str = "\\") -> str:
    """StringUtils.escapeLikeRegex over code points; raises LikePatternError with the reference's error class."""
    out, i = [], 0
    while i < len(pattern):
        c = pattern[i]
        if c == escape and i + 1 < len(pattern):
            c2 = pattern[i + 1]
            if c2 not in ("_", "%", escape):
                raise LikePatternError("INVALID_FORMAT.ESC_IN_THE_MIDDLE")
            out.append(re.escape(c2))
            i += 2
            continue
        if c == escape:
            raise LikePatternError("INVALID_FORMAT.ESC_AT_THE_END")
        out.append("." if c == "_" else ".*" if c == "%" else re.escape(c))
        i += 1
    return "".join(out)


def like(value, pattern: str, escape: str = "\\"):
    """value LIKE pattern ESCAPE escape; value: str, bytes (valid UTF-8) or None."""
    rx = re.compile(like_regex(pattern, escape), re.DOTALL)
    if value is None:
        return None
    if isinstance(value, bytes):
        value = value.decode("utf-8")
    return rx.fullmatch(value) is not None


def _bytes_of(table, name):
    arr = table.column(name)
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    return arr.cast(pa.binary()).to_pylist()


def _lit_bytes(x):
    v = x[1]
    return v if isinstance(v, bytes) else v.encode("utf-8")


def string_test(e, table):
    """(values ndarray, valid bool ndarray) of one string test."""
    op = e[0]
    if op == "str_cmp":
        col_left = e[2][0] == "col"
        name = e[2][1] if col_left else e[3][1]
        lit = _lit_bytes(e[3] if col_left else e[2])
        cmp = {"eq": lambda c: c == 0, "lt": lambda c: c < 0, "le": lambda c: c <= 0, "gt": lambda c: c > 0, "ge": lambda c: c >= 0}[e[1]]
        fn = (lambda s: cmp(O.binary_compare(s, lit))) if col_left else (lambda s: cmp(O.binary_compare(lit, s)))
    else:
        name = e[1][1]
        if op == "in":
            vals = [v for v in e[2] if v is not None]
            has_null = len(vals) != len(e[2])
            fn = lambda s: True if s in vals else (None if has_null else False)          # noqa: E731
        elif op == "starts_with":
            fn = lambda s: s.startswith(e[2])                                             # noqa: E731
        elif op == "ends_with":
            fn = lambda s: s.endswith(e[2])                                               # noqa: E731
        elif op == "contains":
            fn = lambda s: e[2] in s                                                      # noqa: E731
        elif op == "like":
            rx = re.compile(like_regex(e[2], e[3]), re.DOTALL)
            fn = lambda s: rx.fullmatch(s.decode("utf-8")) is not None                    # noqa: E731
        elif op == "octet_length":
            fn = len
        else:
            raise ValueError(op)
    res = [None if s is None else fn(s) for s in _bytes_of(table, name)]
    valid = np.array([r is not None for r in res], bool)
    dt = np.int32 if op == "octet_length" else bool
    return np.array([0 if r is None else r for r in res], dt), valid


def eval_expr(e, table):
    extra = {}

    def sub(x):
        if not isinstance(x, tuple):
            return x
        if x[0] in STRING_OPS:
            v, valid = string_test(x, table)
            name = "__string_test_%d" % len(extra)
            extra[name] = pa.array(v, mask=~valid)
            return ("col", name)
        return tuple(sub(c) for c in x)

    e2 = sub(e)
    t2 = table
    for name, arr in extra.items():
        t2 = t2.append_column(name, arr)
    return O.eval_expr(e2, t2)


def filter_mask(table, predicate):
    v, valid = eval_expr(predicate, table)
    return v.astype(bool) & valid
