"""The CPU restatement of the string-producing functions (tests/string_functions_oracle.py) against the vectors of the reference's
suites (tests/golden/string_functions.json), its stepping over ill-formed UTF-8, and the lowering of the Python expressions."""
import json
import os

import pytest

import string_functions_oracle as O

_GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "string_functions.json")


def _b(x):
    """a golden string: UTF-8 text, {"hex": ...} for raw bytes, or None"""
    if isinstance(x, dict):
        return bytes.fromhex(x["hex"])
    return None if x is None else x.encode("utf-8")


def _vectors():
    with open(_GOLDEN, encoding="utf-8") as f:
        return json.load(f)["vectors"]


def golden_call(v):
    a = v["args"]
    fn = v["fn"]
    if fn == "concat":
        return O.concat(*map(_b, a))
    if fn == "concat_ws":
        return O.concat_ws(*map(_b, a))
    if fn in ("trim", "ltrim", "rtrim"):
        f = getattr(O, fn)
        return f(_b(a[0])) if len(a) == 1 else f(_b(a[0]), _b(a[1]))
    if fn in ("lpad", "rpad"):
        return getattr(O, fn)(_b(a[0]), a[1], _b(a[2]))
    if fn == "substring":
        return O.substring_sql(_b(a[0]), a[1], a[2])
    if fn == "length":
        return O.length(_b(a[0]))
    raise KeyError(fn)


@pytest.mark.parametrize("v", _vectors(), ids=lambda v: "%s-%s" % (v["fn"], v["src"].rsplit("/", 1)[-1]))
def test_golden(v):
    want = v["expect"]
    got = golden_call(v)
    assert got == (want if v["fn"] == "length" else _b(want)), v


def test_golden_cites_every_vector():
    vs = _vectors()
    assert len(vs) > 150
    assert {v["src"].rsplit(":", 1)[1] for v in vs if any(isinstance(a, dict) for a in v["args"])} == {"1362", "1363", "1368"}
    assert all(":" in v["src"] and ("UTF8StringSuite.java" in v["src"] or "StringExpressionsSuite.scala" in v["src"]) for v in vs)
    assert {v["fn"] for v in vs} == {"concat", "concat_ws", "trim", "ltrim", "rtrim", "lpad", "rpad", "substring", "length"}


def test_ill_formed_stepping():
    # a lone continuation byte is one code point; a lead byte declares its width even over ASCII that follows
    assert O.num_chars(b"\x80\x80a") == 3
    assert O.num_chars(b"\xe4a") == 1                 # 0xE4 steps 3 bytes, past the end
    assert O.num_chars(b"\xc0\xc1\xf5\xff") == 4      # bytes no UTF-8 lead allows step by 1
    assert O.substring_sql(b"\xe4ab", 2, 1) == b""
    assert O.substring_sql(b"a\xe4", 2, 5) == b"\xe4"  # truncated at the value's end
    assert O.lpad(b"\xe4a", 3, b"x") == b"xx\xe4a"
    assert O.trim(b"\xa9x\xa9", b"\xc3\xa9") == b"x"  # a lone continuation byte occurs inside the set's bytes


def test_edges():
    assert O.substring_sql(b"abc", 2 ** 31 - 1, 2 ** 31 - 1) == b""
    assert O.substring_sql(b"abc", -2 ** 31, 2 ** 31 - 1) == b"ab"     # start = 3 - 2^31, until = start + len = 2
    assert O.substring_sql(b"abc", -1, 2 ** 31 - 1) == b"c"
    assert O.substring_sql(b"abc", -5, 3) == b"a"
    assert O.lpad(b"ab", -2 ** 31, b"x") == b""
    assert O.rpad(b"ab", 5, b"") == b"ab"
    assert O.concat_ws(b"-", None, None) == b""


def test_lowering():
    from spark_b200 import _capi as capi
    from spark_b200.expressions import (CompiledStringProgram, Concat, ConcatWs, Length, Literal, Schema, StringLPad, StringTrim, Substring,
                                        col)
    schema = Schema(["a", "b", "x"], [capi.SB_STRING, capi.SB_STRING, capi.SB_INT32])
    e = Concat(Substring(col("a"), 1, 2), "-", StringTrim(col("b"), "xy"), StringLPad(col("a"), 5, "0"))
    p = CompiledStringProgram(e, schema)
    op = capi.SB_OP
    got = [(p.arr[i].op, p.arr[i].arg, p.arr[i].arg2) for i in range(p.c.n)]
    assert got == [(op["SF_COL"], 0, 0), (op["SF_SUBSTRING"], 1, 2), (op["SF_LIT"], 0, 0), (op["SF_COL"], 1, 0), (op["SF_TRIM"], 1, 0),
                   (op["SF_COL"], 0, 0), (op["SF_LPAD"], 5, 0), (op["SF_CONCAT"], 4, 0)]
    assert bytes(p.pool)[:p.c.nbytes] == b"-xy0" and p.c.out_type == capi.SB_STRING
    # NULL literal arguments fold to a NULL string
    assert CompiledStringProgram(Substring(col("a"), None, 2), schema).arr[0].arg2 == 1
    assert CompiledStringProgram(ConcatWs(None, col("a")), schema).arr[0].op == op["SF_LIT"]
    with pytest.raises(capi.SparkB200Error) as ei:
        Substring(col("a"), col("x"), 2)
    assert ei.value.code == 5
    with pytest.raises(capi.SparkB200Error):
        StringLPad(col("a"), 5, col("b"))
    from spark_b200.expressions import CompiledExpr
    assert CompiledExpr(Length(col("a")), schema).arr[0].op == op["STR_CHAR_LENGTH"]
    # Length over a binary column is its byte count (Spark's Length over BinaryType)
    bschema = Schema(["a"], [capi.SB_STRING], binary={"a"})
    assert CompiledExpr(Length(col("a")), bschema).arr[0].op == op["STR_OCTET_LENGTH"]
    with pytest.raises(TypeError):
        CompiledExpr(Length(Substring(col("a"), 1, 2)), schema)
