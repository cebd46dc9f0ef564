"""The string-test oracle (tests/string_oracle.py) against the reference's own answers (tests/golden/string_predicates.json:
RegexpExpressionsSuite LIKE, StringExpressionsSuite Contains), and the lowering of the string tests to SB_OP_STR_* programs."""
import json
import os
import struct

import numpy as np
import pyarrow as pa
import pytest

import string_oracle as SO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "string_predicates.json")


def _golden():
    with open(GOLDEN, encoding="utf-8") as f:
        return json.load(f)


@pytest.mark.parametrize("case", _golden()["like"], ids=lambda c: c["source"].rsplit(":", 1)[1])
def test_like_matches_the_reference_vectors(case):
    assert SO.like(case["value"], case["pattern"], case["escape"]) == case["expected"], case


@pytest.mark.parametrize("case", _golden()["like_errors"], ids=lambda c: c["error"])
def test_like_escape_errors(case):
    with pytest.raises(SO.LikePatternError) as ei:
        SO.like(case["value"], case["pattern"], case["escape"])
    assert str(ei.value) == case["error"]


def test_contains_and_the_table_form_match_the_reference_vectors():
    cases = _golden()["contains"]
    t = pa.table({"s": pa.array([c["value"] for c in cases], pa.string())})
    for i, c in enumerate(cases):
        v, valid = SO.eval_expr(("contains", ("col", "s"), c["literal"].encode()), t)
        assert (bool(v[i]) if valid[i] else None) == c["expected"], c
    like = _golden()["like"]
    t = pa.table({"s": pa.array([c["value"] for c in like], pa.string())})
    for i, c in enumerate(like):
        v, valid = SO.eval_expr(("like", ("col", "s"), c["pattern"], c["escape"]), t)
        assert (bool(v[i]) if valid[i] else None) == c["expected"], c


def test_in_comparisons_and_octet_length_over_bytes():
    vals = [b"", b"a", b"ab", b"b", b"\x00", b"\xff", b"a\x00", None, "€".encode()]
    arr = pa.Array.from_buffers(pa.string(), len(vals), [pa.py_buffer(np.packbits([v is not None for v in vals], bitorder="little").tobytes()),
                                                         pa.py_buffer(np.cumsum([0] + [len(v or b"") for v in vals]).astype(np.int32).tobytes()),
                                                         pa.py_buffer(b"".join(v or b"" for v in vals))], null_count=1)
    t = pa.table({"s": arr})

    def run(e):
        v, valid = SO.eval_expr(e, t)
        return [bool(x) if x.dtype == bool else int(x) if ok else None for x, ok in zip(v, valid)] if v.dtype != bool else \
            [bool(x) if ok else None for x, ok in zip(v, valid)]
    assert run(("in", ("col", "s"), [b"a", b"\xff"])) == [False, True, False, False, False, True, False, None, False]
    assert run(("in", ("col", "s"), [b"a", None])) == [None, True, None, None, None, None, None, None, None]
    assert run(("str_cmp", "lt", ("col", "s"), ("lit", b"a", bytes))) == [True, False, False, False, True, False, False, None, False]
    assert run(("str_cmp", "lt", ("lit", b"a", bytes), ("col", "s"))) == [False, False, True, True, False, True, True, None, True]
    assert run(("octet_length", ("col", "s"))) == [0, 1, 2, 1, 1, 1, 2, None, 3]
    assert run(("ends_with", ("col", "s"), b"")) == [True] * 7 + [None, True]
    assert run(("not", ("starts_with", ("col", "s"), b"a"))) == [True, False, False, True, True, True, False, None, True]


def test_string_tests_lower_to_leaves_over_one_pool():
    from spark_b200 import _capi as capi
    from spark_b200.expressions import (CompiledExpr, Contains, EndsWith, In, Like, Literal, OctetLength, Schema, StartsWith, col)
    schema = Schema(["x", "s"], [capi.SB_INT32, capi.SB_STRING])
    e = (Literal("m") < col("s")) & Like(col("s"), "a!%%", escape="!") & In(col("s"), ["bb", None, "a"]) & \
        (OctetLength(col("s")) > Literal(2)) & StartsWith(col("s"), "p") & EndsWith(col("s"), b"\xff") & Contains(col("s"), "") & \
        col("s").eq("BUILDING") & (col("x") > Literal(1))
    ce = CompiledExpr(e, schema)
    nodes = [ce.arr[i] for i in range(ce.c.n)]
    pool = bytes(ce.pool)[:ce.c.nbytes]
    leaves = [(nd.op, nd.vtype, nd.arg, nd.arg2, pool[nd.lit.i >> 32:(nd.lit.i >> 32) + (nd.lit.i & 0xffffffff)]) for nd in nodes
              if nd.op >= capi.SB_OP["STR_EQ"]]
    op = capi.SB_OP
    assert leaves == [(op["STR_GT"], 1, 1, 0, b"m"), (op["STR_LIKE"], 1, 1, ord("!"), b"a!%%"),
                      (op["STR_IN"], 1, 1, 1, struct.pack("=I", 2) + struct.pack("=I", 2) + b"bb" + struct.pack("=I", 1) + b"a"),
                      (op["STR_OCTET_LENGTH"], 2, 1, 0, b""), (op["STR_STARTS_WITH"], 1, 1, 0, b"p"), (op["STR_ENDS_WITH"], 1, 1, 0, b"\xff"),
                      (op["STR_CONTAINS"], 1, 1, 0, b""), (op["STR_EQ"], 1, 1, 0, b"BUILDING")]
    assert all(nd.arg2 == 0 for nd in nodes if nd.op < op["STR_EQ"])
    assert ce.c.out_type == capi.SB_BOOL and CompiledExpr(OctetLength(col("s")), schema).c.out_type == capi.SB_INT32
    plain = CompiledExpr(col("x") > Literal(1), schema)
    assert plain.c.nbytes == 0 and not plain.c.bytes
    with pytest.raises(TypeError):
        CompiledExpr(StartsWith(col("x"), "a"), schema)
