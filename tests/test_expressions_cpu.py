"""Expression semantics without a device: the oracle's evaluator pinned to answers Java and Spark SQL give, and the programs the
Python emitter (spark_b200/expressions.py) lowers expressions to.  The GPU evaluators are checked against this oracle in
tests/test_gpu_expressions.py, so a wrong oracle would make every parity test agree with the wrong answer."""
import struct

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as O

I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1


def _one(e, **cols):
    """Evaluate `e` over a one-row table -> (python value, is valid)."""
    v, valid = O.eval_expr(e, pa.table(cols))
    return v[0].item(), bool(valid[0])


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


D = lambda x: pa.array([x], pa.float64())          # noqa: E731
F = lambda x: pa.array([x], pa.float32())          # noqa: E731
I = lambda x: pa.array([x], pa.int32())            # noqa: E731
L = lambda x: pa.array([x], pa.int64())            # noqa: E731


# JLS 5.1.3 narrowing of double to int / long: NaN -> 0, toward zero, saturating (Cast.scala:1159-1161 runs Java's conversion)
@pytest.mark.parametrize("op,x,want", [
    ("cast_i32", float("nan"), 0), ("cast_i64", float("nan"), 0),
    ("cast_i32", 1e10, 2147483647), ("cast_i32", -1e10, -2147483648), ("cast_i32", -2.9, -2), ("cast_i32", 2.9, 2),
    ("cast_i32", float("inf"), 2147483647), ("cast_i32", float("-inf"), -2147483648), ("cast_i32", -0.0, 0),
    ("cast_i64", 1e19, 9223372036854775807), ("cast_i64", float("-inf"), -9223372036854775808),
    ("cast_i64", float("inf"), 9223372036854775807), ("cast_i64", -2.9, -2), ("cast_i64", 2.0 ** 62, 4611686018427387904),
    ("cast_i64", 9.223372036854775e18, 9223372036854774784),
])
def test_oracle_double_to_integer_casts_follow_java(op, x, want):
    assert _one((op, ("col", "d")), d=D(x)) == (want, True)


def test_oracle_integer_casts_and_widening():
    assert _one(("cast_i32", ("col", "l")), l=L(3000000000)) == (-1294967296, True)          # (int) 3000000000L
    assert _one(("cast_i32", ("col", "l")), l=L(I64_MIN)) == (0, True)
    assert _one(("cast_i64", ("col", "i")), i=I(I32_MIN)) == (I32_MIN, True)
    assert _one(("cast_f64", ("col", "f")), f=F(0.1)) == (0.10000000149011612, True)         # (double) 0.1f
    assert _one(("cast_f64", ("col", "l")), l=L(2 ** 53 + 1)) == (2.0 ** 53, True)            # (double) (2^53 + 1), ties to even
    assert _one(("cast_i64", ("col", "l")), l=pa.array([None], pa.int64()))[1] is False


def test_oracle_integer_arithmetic_wraps_at_the_operand_width():
    assert _one(("add", ("col", "i"), ("lit", 1, np.int32)), i=I(I32_MAX)) == (I32_MIN, True)
    assert _one(("mul", ("col", "i"), ("col", "i")), i=I(46341)) == (-2147479015, True)
    assert _one(("sub", ("col", "i"), ("lit", 1, np.int32)), i=I(I32_MIN)) == (I32_MAX, True)
    assert _one(("neg", ("col", "l")), l=L(I64_MIN)) == (I64_MIN, True)
    assert _one(("neg", ("col", "i")), i=I(I32_MIN)) == (I32_MIN, True)
    assert _one(("add", ("col", "l"), ("lit", 1, np.int64)), l=L(I64_MAX)) == (I64_MIN, True)


def test_oracle_double_arithmetic():
    assert _one(("add", ("col", "d"), ("lit", 0.2, np.float64)), d=D(0.1)) == (0.30000000000000004, True)
    v, ok = _one(("neg", ("col", "d")), d=D(0.0))
    assert ok and _bits(v) == _bits(-0.0)
    for divisor in (0.0, -0.0):                                                              # Divide: NULL on a zero divisor
        assert _one(("div", ("lit", 1.0, np.float64), ("col", "d")), d=D(divisor))[1] is False
    assert _one(("div", ("lit", 1.0, np.float64), ("col", "i")), i=I(0))[1] is False
    v, ok = _one(("div", ("lit", 1.0, np.float64), ("col", "d")), d=D(float("nan")))
    assert ok and v != v


def test_oracle_sql_comparisons_and_three_valued_logic():
    nan, inf = float("nan"), float("inf")
    assert _one(("eq", ("col", "d"), ("lit", nan, np.float64)), d=D(nan)) == (True, True)    # compareDoubles: NaN = NaN
    assert _one(("gt", ("col", "d"), ("lit", inf, np.float64)), d=D(nan)) == (True, True)    # NaN > +inf
    assert _one(("eq", ("col", "d"), ("lit", 0.0, np.float64)), d=D(-0.0)) == (True, True)   # -0.0 = 0.0
    assert _one(("lt", ("col", "d"), ("lit", 0.0, np.float64)), d=D(-0.0)) == (False, True)
    assert _one(("ne", ("col", "d"), ("lit", nan, np.float64)), d=D(1.0)) == (True, True)
    null_bool = ("lit", None, bool)
    assert _one(("and", null_bool, ("lit", False, bool)), i=I(0)) == (False, True)            # NULL AND false = false
    assert _one(("and", null_bool, ("lit", True, bool)), i=I(0))[1] is False                # NULL AND true = NULL
    assert _one(("or", null_bool, ("lit", True, bool)), i=I(0)) == (True, True)              # NULL OR true = true
    assert _one(("or", null_bool, ("lit", False, bool)), i=I(0))[1] is False
    assert _one(("not", null_bool), i=I(0))[1] is False                                     # NOT NULL = NULL
    assert _one(("lt", ("col", "i"), ("lit", None, np.int32)), i=I(1))[1] is False           # a comparison with NULL is NULL
    assert _one(("isnull", ("lit", None, np.int64)), i=I(0)) == (True, True)


def test_float32_is_evaluated_in_double_and_one_rounding_matches_java():
    """float32 operands are widened and evaluated in double (DESIGN §2).  One add / sub / mul / div rounded back to float is Java's
    float result (53 >= 2 * 24 + 2 makes the double rounding harmless); a chain of two operations can differ."""
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(20000) * np.exp2(rng.integers(-30, 30, 20000))).astype(np.float32)
    b = (rng.standard_normal(20000) * np.exp2(rng.integers(-30, 30, 20000))).astype(np.float32)
    with np.errstate(all="ignore"):
        for f in (np.add, np.subtract, np.multiply, np.divide):
            via_double = f(a.astype(np.float64), b.astype(np.float64)).astype(np.float32)
            assert np.array_equal(via_double.view(np.int32), f(a, b).view(np.int32)), f
    one, tiny = np.float32(1.0), np.float32(2.0 ** -24)
    assert (one + tiny) + tiny == one                                                     # float chain: both adds round away
    assert np.float32((np.float64(one) + tiny) + tiny) == np.float32(1.0 + 2.0 ** -23)     # double chain keeps them


# ---- the Python emitter's programs --------------------------------------------------------------------------------------------
def _programs():
    from spark_b200 import _capi as capi
    from spark_b200.expressions import Cast, Divide, Literal, Schema, col
    names = ["b", "i8", "i16", "i32", "dt", "i64", "ts", "f32", "f64"]
    schema = Schema(names, [capi.SB_BOOL, capi.SB_INT8, capi.SB_INT16, capi.SB_INT32, capi.SB_DATE32, capi.SB_INT64, capi.SB_TIMESTAMP,
                            capi.SB_FLOAT32, capi.SB_FLOAT64])
    exprs = []
    for x in names:
        for y in names:
            exprs += [col(x) < col(y), col(x).eq(col(y)), col(x).ne(col(y))]
            if x != "b" and y != "b":
                exprs += [col(x) + col(y), col(x) * col(y) - col(x), Divide(col(x), col(y))]
        for lit in (Literal(1), Literal(2 ** 40), Literal(0.5), Literal(None), Literal(True)):
            exprs += [col(x) >= lit, lit > col(x), col(x).eq(lit)]
        for to in ("int", "long", "double"):
            exprs += [Cast(col(x), to), Cast(col(x), to) > Literal(0), Cast(Cast(col(x), to), "double") + Literal(1)]
        exprs += [-col(x) if x != "b" else ~col(x), col(x).is_null(), ~(col(x) < Literal(3)) | col(x).is_not_null()]
    exprs += [Literal(None) + col("i32"), Literal(None) * col("f64"), (Literal(1) - col("f64")) * (col("f32") + Literal(1))]
    return schema, exprs


def test_emitter_casts_and_comparisons_carry_their_operand_class():
    """Every implicit coercion is a CAST whose `arg` is the class of the value it converts, and a comparison's `arg` is the class of
    both its operands: the kernels read the source class from `arg` and would otherwise reinterpret the bits."""
    from spark_b200 import _capi as capi
    from spark_b200.expressions import CompiledExpr
    ops = {v: k for k, v in capi.SB_OP.items()}
    schema, exprs = _programs()
    n_cast = n_cmp = 0
    for e in exprs:
        ce = CompiledExpr(e, schema)
        stack = []
        for i in range(ce.c.n):
            nd = ce.arr[i]
            op = ops[nd.op]
            if op in ("COL", "LIT_I64", "LIT_F64", "LIT_NULL"):
                stack.append(nd.vtype)
                continue
            if op in ("NEG", "NOT", "ISNULL", "ISNOTNULL", "CAST_F64", "CAST_I64", "CAST_I32"):
                src = stack.pop()
                if op.startswith("CAST"):
                    n_cast += 1
                    assert nd.arg == src, (e.sexpr(), i, nd.arg, src)
                    assert nd.vtype == {"CAST_F64": capi.SB_VT_F64, "CAST_I64": capi.SB_VT_I64, "CAST_I32": capi.SB_VT_I32}[op]
                    assert src != nd.vtype, "a cast to the operand's own class is emitted as nothing"
                stack.append(nd.vtype)
                continue
            r, l = stack.pop(), stack.pop()
            if op in ("EQ", "NE", "LT", "LE", "GT", "GE"):
                n_cmp += 1
                assert l == r == nd.arg, (e.sexpr(), i, l, r, nd.arg)
                assert nd.vtype == capi.SB_VT_BOOL
            elif op in ("ADD", "SUB", "MUL", "DIV"):
                assert l == r == nd.vtype, (e.sexpr(), i, l, r, nd.vtype)
            stack.append(nd.vtype)
        assert len(stack) == 1
    assert n_cast > 100 and n_cmp > 200
