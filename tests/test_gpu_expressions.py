"""Every GPU evaluator of expression programs, bit for bit against the oracle, at the edges of each type.

Six pieces of code evaluate sb_expr programs (include/spark_b200.h SB_OP_*): the interpreter (csrc/expr.cu eval_row), the typed
16-rows-per-thread filter (simple_pred_eval16), the lane-strided filter inside the join's candidate pass (simple_pred_rows), the
aggregate's fused filter terms and fused products (csrc/agg_kernels.cuh), and the host matchers choosing between them.  Each test
isolates one evaluator's per-row verdicts or values on one adversarial table: MIN / MAX / -1 / 0 / 1 of every integer width,
+-inf, +-0.0, NaNs with payloads and sign bits, subnormals, 2^53 + 1, 0.1f, NULLs.

util.assert_tables_equal allows 1e-6 and treats -0.0 as 0.0, so values are compared here by bit pattern (any NaN for a NaN)."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as O
from spark_b200.expressions import Expression, _node      # host-side only: importing loads no library

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
NAN, INF = float("nan"), float("inf")
NAN_PAYLOAD = 0x7FF8000000000123                     # quiet NaN with payload bits (as LIT_F64 bits)
F64_SPECIAL = [0x7FF0000000000000, 0xFFF0000000000000, 0, 0x8000000000000000, 0x7FF8000000000000, NAN_PAYLOAD,
               0xFFF8000000000000, 0x7FF0000000000001, 1, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF]
F64_SPECIAL_VALUES = [0.1, 2.0 ** 53, 2.0 ** 53 + 2, 1.0, -1.0, 0.5, -2.5, 1e10, -1e19, 2.9, -2.9]
F32_SPECIAL = [0x7F800000, 0xFF800000, 0, 0x80000000, 0x7FC00000, 0x7FC00123, 0xFFC00000, 0x00000001, 0x7F7FFFFF]
F32_SPECIAL_VALUES = [0.1, 1.0, -1.0, 0.5, 3e9, -2.5]
INT_RANGE = {"i8": 8, "i16": 16, "i32": 32, "dt": 32, "i64": 64, "ts": 64}
NP_OF = {"i8": np.int8, "i16": np.int16, "i32": np.int32, "dt": np.int32, "i64": np.int64, "ts": np.int64}


def _specials_int(name):
    b = INT_RANGE[name]
    lo, hi = -2 ** (b - 1), 2 ** (b - 1) - 1
    s = [lo, hi, -1, 0, 1, lo + 1, hi - 1]
    if b == 64:
        s += [2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 31, -2 ** 31 - 1, 3000000000]
    return np.array(s, dtype=NP_OF[name])


def _f64_specials():
    return np.concatenate([np.array(F64_SPECIAL, np.uint64).view(np.float64), np.array(F64_SPECIAL_VALUES)])


def _f32_specials():
    return np.concatenate([np.array(F32_SPECIAL, np.uint32).view(np.float32), np.array(F32_SPECIAL_VALUES, np.float32)])


def _mix(rng, n, specials, filler):
    v = filler.copy()
    pick = rng.random(n) < 0.35
    v[pick] = specials[rng.integers(0, len(specials), int(pick.sum()))]
    return v


def adversarial_table(n, seed, nullable=True):
    """Columns b, i8, i16, i32, dt, i64, ts, f32, f64, g64, h64 (edge values + small random filler, NULLs in all but i16 and h64),
    g (row % 7) and row (0..n-1)."""
    rng = np.random.default_rng(seed)
    mask = (lambda: rng.random(n) < 0.15) if nullable else (lambda: None)
    cols = {"b": pa.array(rng.random(n) < 0.5, mask=mask())}
    for name in ("i8", "i16", "i32", "dt", "i64", "ts"):
        filler = rng.integers(-3, 4, n).astype(NP_OF[name])
        v = _mix(rng, n, _specials_int(name), filler)
        m = None if name == "i16" else mask()
        arr = pa.array(v, mask=m)
        if name == "dt":
            arr = arr.cast(pa.date32())
        elif name == "ts":
            arr = arr.cast(pa.timestamp("us"))
        cols[name] = arr
    small = np.array([-1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0, 0.1, 3.0])
    f32 = _mix(rng, n, _f32_specials(), np.where(rng.random(n) < 0.5, small[rng.integers(0, len(small), n)],
                                                 rng.standard_normal(n) * 10).astype(np.float32))
    cols["f32"] = pa.array(f32, mask=mask())
    for name in ("f64", "g64", "h64"):
        f = _mix(rng, n, _f64_specials(), np.where(rng.random(n) < 0.5, small[rng.integers(0, len(small), n)], rng.standard_normal(n) * 10))
        cols[name] = pa.array(f, mask=None if name == "h64" else mask())
    cols["g"] = (np.arange(n) % 7).astype(np.int32)
    cols["row"] = np.arange(n, dtype=np.int64)
    return pa.table(cols)


# ---- bit-exact comparison -----------------------------------------------------------------------------------------------------
def _host(arr):
    """(values, valid) of an arrow column as numpy, values read from the data buffer (bit patterns kept)."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    n = len(arr)
    valid = np.ones(n, bool) if arr.null_count == 0 else np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), bool)
    t = arr.type
    if pa.types.is_boolean(t):
        return np.asarray(arr.fill_null(False).to_numpy(zero_copy_only=False), bool), valid
    if pa.types.is_date32(t):
        dt = np.int32
    elif pa.types.is_timestamp(t):
        dt = np.int64
    else:
        dt = t.to_pandas_dtype()
    return np.frombuffer(arr.buffers()[1], dtype=dt)[arr.offset:arr.offset + n], valid


def assert_bits(got, want, what):
    """`got`: arrow column from the GPU; `want`: (values, valid) from oracle.eval_expr.  NULLs must agree; integers and booleans
    compare exactly, doubles by bit pattern (float32 oracle values are widened first, which is exact), any NaN matching a NaN."""
    gv, gm = _host(got)
    wv, wm = want
    wm = np.asarray(wm, bool)
    bad = np.flatnonzero(gm != wm)
    assert len(bad) == 0, "%s: NULL mismatch at rows %s (got valid %s)" % (what, bad[:8], gm[bad[:8]])
    gv, wv = gv[wm], np.asarray(wv)[wm]
    if gv.dtype.kind == "f" or wv.dtype.kind == "f":
        assert gv.dtype.kind == "f" and wv.dtype.kind == "f", (what, gv.dtype, wv.dtype)
        g, w = gv.astype(np.float64), wv.astype(np.float64)
        ok = (g.view(np.int64) == w.view(np.int64)) | (np.isnan(g) & np.isnan(w))
    else:
        g, w = gv.astype(np.int64), wv.astype(np.int64)
        ok = g == w
    bad = np.flatnonzero(~ok)
    assert len(bad) == 0, "%s: %d values differ, first at valid row %d: got %r want %r" % (what, len(bad), bad[0], g[bad[0]], w[bad[0]])


# ---- hand-built programs: what the Python sugar never emits -------------------------------------------------------------------
VT = {"b": 1, "i8": 2, "i16": 2, "i32": 2, "dt": 2, "i64": 3, "ts": 3, "f32": 4, "f64": 4, "g64": 4, "h64": 4, "g": 2, "row": 3}
NP_OF_VT = {1: bool, 2: np.int32, 3: np.int64, 4: np.float64}


class Raw(Expression):
    """A hand-built postfix program.  nodes: (op, vtype, arg, lit); a COL's arg is a column name, an int lit of a LIT_F64 is its
    bit pattern."""

    def __init__(self, nodes, sexpr=None, vt=1):
        self.nodes, self._sexpr, self.vt = nodes, sexpr, vt

    def vtype(self, schema):
        return self.vt

    def emit(self, schema, out):
        for op, vt, arg, lit in self.nodes:
            out.append(_node(op, vt, schema.index(arg) if op == "COL" else arg,
                             lit_i=lit if isinstance(lit, int) else None, lit_d=lit if isinstance(lit, float) else None))

    def sexpr(self):
        return self._sexpr

    def references(self):
        return {a for op, _, a, _ in self.nodes if op == "COL"}


def _col(name):
    return ("COL", VT[name], name, None)


def _lit(vt, v):
    if v is None:
        return ("LIT_NULL", vt, 0, None)
    return ("LIT_F64", 4, 0, v) if vt == 4 else ("LIT_I64", vt, 0, int(v))


def _lit_sexpr(vt, v):
    if isinstance(v, int) and vt == 4:           # NaN given by its bits
        v = float(np.array([v], np.uint64).view(np.float64)[0])
    return ("lit", v, NP_OF_VT[vt])


def raw_compare(op, name, v, lit_left=False):
    """`name <op> v` (or `v <op> name`) as a raw program; v None is a NULL literal of the column's class."""
    vt = VT[name]
    c, l = _col(name), _lit(vt, v)
    lhs, rhs = (l, c) if lit_left else (c, l)
    s_c, s_l = ("col", name), _lit_sexpr(vt, v)
    return Raw([lhs, rhs, (op.upper(), 1, vt, None)], (op, s_l, s_c) if lit_left else (op, s_c, s_l))


def raw_and(*terms):
    nodes, s = list(terms[0].nodes), terms[0].sexpr()
    for t in terms[1:]:
        nodes += t.nodes + [("AND", 1, 0, None)]
        s = ("and", s, t.sexpr())
    return Raw(nodes, s)


# ---- literals per column ------------------------------------------------------------------------------------------------------
LITERALS = {"b": [True, False], "i8": [-128, 127, 0, -1], "i16": [-32768, 32767, 1], "i32": [I32_MIN, I32_MAX, 0, -1],
            "dt": [I32_MIN, 0, 1], "i64": [I64_MIN, I64_MAX, 0, 2 ** 53 + 1], "ts": [I64_MIN, -1, 1],
            "f32": [0.1, -0.0, NAN, INF, 1.401298464324817e-45, 1.0], "f64": [NAN, -0.0, INF, -INF, 5e-324, 0.1, 2.0 ** 53]}


def _py_literal(name, v):
    from spark_b200.expressions import Literal
    return Literal(v, {1: 1, 2: 2, 3: 3, 4: 4}[VT[name]])


def filter_conditions():
    """Every comparison against every column type, literal on either side (SB_OP_NE hand-built), 4- and 5-term conjunctions,
    NULL literals of every class inside comparisons, arithmetic and Kleene logic."""
    from spark_b200.expressions import (EqualTo, GreaterThan, GreaterThanOrEqual, LessThan, LessThanOrEqual, Literal, col)
    ops = [LessThan, LessThanOrEqual, GreaterThan, GreaterThanOrEqual, EqualTo]
    conds = []
    for name, lits in LITERALS.items():
        for v in lits:
            lit = _py_literal(name, v)
            for op in ops:
                conds += [op(col(name), lit), op(lit, col(name))]
            conds += [raw_compare("ne", name, v), raw_compare("ne", name, v, lit_left=True)]
    conds.append(raw_compare("eq", "f64", NAN_PAYLOAD))
    conds.append(raw_compare("ne", "f64", NAN_PAYLOAD))
    four = [(col("f64") > Literal(0.0)), (col("i32") >= Literal(-1)), (col("f32") <= Literal(1.0)), col("i64").is_not_null()]
    conds.append(four[0] & four[1] & four[2] & four[3])
    conds.append((col("b").eq(Literal(True))) & (col("dt") < Literal(2)) & (col("ts") >= Literal(-1)) & (col("i16") > Literal(-2)))
    conds.append(four[0] & four[1] & four[2] & four[3] & (col("i8") < Literal(1)))                       # 5 terms: interpreter
    conds.append(raw_and(raw_compare("ne", "f64", NAN), raw_compare("ne", "i32", 0), raw_compare("lt", "f32", NAN, True)))
    conds.append(col("f32").is_not_null())
    for name in ("b", "i32", "i64", "f64", "f32"):
        vt = VT[name]
        conds.append(raw_compare("lt", name, None))
        conds.append(raw_compare("ge", name, None, lit_left=True))
        conds.append(Raw([_col(name), _lit(vt, None), ("LT", 1, vt, None), ("NOT", 1, 0, None)],
                         ("not", ("lt", ("col", name), _lit_sexpr(vt, None)))))
        conds.append(Raw([_col(name), _lit(vt, None), ("EQ", 1, vt, None), _col(name), _lit(vt, 0 if vt < 4 else 0.0), ("GE", 1, vt, None),
                          ("OR", 1, 0, None)],
                         ("or", ("eq", ("col", name), _lit_sexpr(vt, None)), ("ge", ("col", name), _lit_sexpr(vt, 0 if vt < 4 else 0.0)))))
    for name in ("i32", "i64", "f64"):
        vt = VT[name]
        zero = 0 if vt < 4 else 0.0
        conds.append(Raw([_col(name), _lit(vt, None), ("ADD", vt, 0, None), _lit(vt, zero), ("GT", 1, vt, None)],
                         ("gt", ("add", ("col", name), _lit_sexpr(vt, None)), _lit_sexpr(vt, zero))))
        conds.append(Raw([_lit(vt, None), _col(name), ("MUL", vt, 0, None), _lit(vt, zero), ("LE", 1, vt, None), _col(name), _lit(vt, zero),
                          ("LT", 1, vt, None), ("OR", 1, 0, None)],
                         ("or", ("le", ("mul", _lit_sexpr(vt, None), ("col", name)), _lit_sexpr(vt, zero)), ("lt", ("col", name), _lit_sexpr(vt, zero)))))
    conds.append(Raw([_lit(1, None), ("NOT", 1, 0, None), _col("i32"), _lit(2, 0), ("GT", 1, 2, None), ("OR", 1, 0, None)],
                     ("or", ("not", ("lit", None, bool)), ("gt", ("col", "i32"), ("lit", 0, np.int32)))))
    return conds


def _scan(t, stream):
    from spark_b200.columnar import ColumnarBatch
    return ColumnarBatch.from_arrow(t, stream)


@pytest.mark.parametrize("interpret_only", [False, True], ids=["typed-fast-path", "interpreter"])
@pytest.mark.parametrize("n", [1, 15, 16, 17, 25, 4097, 100_003])
def test_filter_verdicts_at_the_edges_of_every_type(gpu, stream, n, interpret_only, sbconfig):
    """FilterExec keeps exactly the rows whose predicate is TRUE.  At n = 25 the last 16-row group has 9 rows: its last row's
    validity lives in the group's second bitmap byte."""
    from spark_b200.execution import FilterExec, LocalTableScanExec, ProjectExec
    sbconfig("expr_interpret_only", 1 if interpret_only else 0)
    t = adversarial_table(n, seed=n)
    batch = _scan(t, stream)
    try:
        for cond in filter_conditions():
            got = ProjectExec(["row"], FilterExec(cond, LocalTableScanExec(batch))).collect(stream)
            want = O.filter_table(t, cond.sexpr())
            g, w = np.asarray(got.column("row")), np.asarray(want.column("row"))
            assert np.array_equal(g, w), (cond.sexpr(), np.setdiff1d(g, w)[:5], np.setdiff1d(w, g)[:5])
    finally:
        batch.close()


def projections():
    from spark_b200.expressions import Cast, Divide, Literal, UnaryMinus, col
    p = []
    for x, y in (("i32", "i32"), ("i64", "i64"), ("i32", "i64"), ("f64", "g64"), ("f64", "f32"), ("i64", "f64")):
        p += [col(x) + col(y), col(x) - col(y), col(x) * col(y)]
    p += [UnaryMinus(col(c)) for c in ("i32", "i64", "f64", "f32")]
    p += [col("i32") + Literal(1), Literal(I32_MIN) - col("i32"), col("i64") * Literal(-1), Literal(I64_MAX) + col("i64"),
          col("f64") * Literal(0.1) + Literal(0.2)]
    p += [Divide(col("f64"), col("g64")), Divide(col("i32"), col("i64")), Divide(col("f64"), Literal(0.0)), Divide(col("f64"), Literal(-0.0)),
          Divide(col("f64"), Literal(NAN)), Divide(Literal(1.0), col("i32")), Divide(col("f32"), col("f64"))]
    for c in ("b", "i8", "i32", "i64", "f32", "f64"):
        p += [Cast(col(c), "int"), Cast(col(c), "long"), Cast(col(c), "double")]
    p += [Cast(col("f64") * Literal(1e10), "int"), Cast(Cast(col("i64"), "double"), "long")]
    for c in ("b", "i8", "i16", "i32", "dt", "i64", "ts", "f32", "f64"):
        p += [col(c).is_null(), col(c).is_not_null()]
    p += [~col("b"), ~Literal(None), Literal(None) & (col("i32") < Literal(0)), Literal(None) | (col("i32") < Literal(0)),
          ~(col("f64") > Literal(0.0)), col("b") | (col("f64") < Literal(NAN)), col("b") & col("f64").is_null()]
    p.append(Raw([_lit(4, 0.0), ("NEG", 4, 0, None)], ("neg", ("lit", 0.0, np.float64)), vt=4))                  # -(0.0) = -0.0
    for vt in (2, 3, 4):
        name = {2: "i32", 3: "i64", 4: "f64"}[vt]
        p.append(Raw([_col(name), _lit(vt, None), ("SUB", vt, 0, None)], ("sub", ("col", name), _lit_sexpr(vt, None)), vt=vt))
        p.append(Raw([_lit(vt, None), ("NEG", vt, 0, None)], ("neg", _lit_sexpr(vt, None)), vt=vt))
    deep = [_lit(2, 1)] * 12 + [("ADD", 2, 0, None)] * 11                      # exactly EXPR_STACK slots
    s = ("lit", 1, np.int32)
    for _ in range(11):
        s = ("add", ("lit", 1, np.int32), s)
    p.append(Raw(deep, s, vt=2))
    return p


@pytest.mark.parametrize("n", [25, 100_003])
@pytest.mark.parametrize("filtered", [False, True], ids=["all-rows", "below-a-filter"])
def test_projection_values_are_bit_exact(gpu, stream, n, filtered):
    """ProjectExec: wrapping integer arithmetic, -x of MIN, double arithmetic on +-0 / inf / NaN, Divide by 0, -0.0 and NaN, every
    cast from every class (Java's saturating double -> int / long), IS [NOT] NULL, NOT / AND / OR over NULL."""
    from spark_b200.execution import FilterExec, LocalTableScanExec, ProjectExec
    from spark_b200.expressions import Literal, col
    t = adversarial_table(n, seed=7 + n)
    cond = col("i16") >= Literal(0)
    src = O.filter_table(t, cond.sexpr()) if filtered else t
    exprs = projections()
    batch = _scan(t, stream)
    try:
        plan = ProjectExec([("p%d" % i, e) for i, e in enumerate(exprs)], FilterExec(cond, LocalTableScanExec(batch)) if filtered else LocalTableScanExec(batch))
        got = plan.collect(stream)
    finally:
        batch.close()
    assert got.num_rows == src.num_rows
    for i, e in enumerate(exprs):
        assert_bits(got.column("p%d" % i), O.eval_expr(e.sexpr(), src), e.sexpr())


def test_documented_deviations_are_pinned(gpu, stream):
    """DESIGN §2: tinyint / smallint arithmetic is evaluated at 32 bits (Spark wraps at the operand width), and float32 operands are
    evaluated in double: one operation rounded back to float is Java's float result, a chain of two can differ."""
    from spark_b200.execution import LocalTableScanExec, ProjectExec
    from spark_b200.expressions import col
    t = pa.table({"a": np.array([127, -128, 100], np.int8), "s": np.array([32767, -32768, 1], np.int16)})
    batch = _scan(t, stream)
    try:
        got = ProjectExec([("x", col("a") + col("a")), ("y", col("s") * col("s"))], LocalTableScanExec(batch)).collect(stream)
    finally:
        batch.close()
    assert got.column("x").to_pylist() == [254, -256, 200]
    assert O.eval_expr(("add", ("col", "a"), ("col", "a")), t)[0].tolist() == [-2, 0, -56]          # what Spark returns
    assert got.column("y").to_pylist() == [1073676289, 1073741824, 1]
    rng = np.random.default_rng(3)
    n = 50_000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    a[:3], b[:3] = np.float32(1.0), np.float32(2.0 ** -24)
    batch = _scan(pa.table({"a": a, "b": b}), stream)
    try:
        got = ProjectExec([("add", col("a") + col("b")), ("sub", col("a") - col("b")), ("mul", col("a") * col("b")), ("div", col("a") / col("b")),
                           ("chain", col("a") + col("b") + col("b"))], LocalTableScanExec(batch)).collect(stream)
    finally:
        batch.close()
    for name, f in (("add", np.add), ("sub", np.subtract), ("mul", np.multiply), ("div", np.divide)):
        g = np.asarray(got.column(name)).astype(np.float32)
        assert np.array_equal(g.view(np.int32), f(a, b).view(np.int32)), name
    chain = np.asarray(got.column("chain")).astype(np.float32)
    assert chain[0] == np.float32(1.0 + 2.0 ** -23) and (a[0] + b[0]) + b[0] == np.float32(1.0)   # Java's float chain rounds twice


# ---- joins --------------------------------------------------------------------------------------------------------------------
def join_probe_conditions():
    from spark_b200.expressions import EqualTo, GreaterThan, Literal, col
    return [(col("f64") > Literal(0.0)) & (col("i32") >= Literal(-1)),
            (col("f32") < Literal(1.0)) & (col("dt") <= Literal(0)),
            EqualTo(col("f64"), Literal(NAN)) & col("b").eq(Literal(True)),
            (col("i8") > Literal(-128)) & (col("i16") < Literal(32767)) & (col("ts") >= Literal(0)) & col("i64").is_not_null(),
            GreaterThan(Literal(NAN), col("f32")) & (col("i32") < Literal(I32_MAX)) & (col("i64") <= Literal(2 ** 53 + 1)),
            raw_and(raw_compare("ne", "f64", NAN_PAYLOAD), raw_compare("ne", "i32", 0), raw_compare("gt", "g64", -0.0, True)),
            (col("f64") <= Literal(-0.0)) & (col("g64") >= Literal(5e-324))]


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
def test_join_probe_filter_in_the_candidate_pass(gpu, stream, variant, sbconfig):
    """A left semi join whose relation holds every key: its output rows are exactly the streamed FilterExec's verdicts, evaluated
    inside the candidate pass (2^20 + ragged streamed rows) by every pass variant."""
    from spark_b200.execution import BroadcastHashJoinExec, FilterExec, LocalTableScanExec
    sbconfig("join_cand", variant)
    n, nb = (1 << 20) + 4099, 4096
    t = adversarial_table(n, seed=41)
    t = t.append_column("fk", pa.array(np.arange(n, dtype=np.int64) % nb))
    build = pa.table({"id": np.arange(nb, dtype=np.int64)})
    pb, bb = _scan(t, stream), _scan(build, stream)
    try:
        for cond in join_probe_conditions():
            got = BroadcastHashJoinExec(["fk"], ["id"], "left_semi", "right", FilterExec(cond, LocalTableScanExec(pb)),
                                        LocalTableScanExec(bb)).collect(stream)
            want = np.flatnonzero(O.filter_mask(t, cond.sexpr()))
            g = np.asarray(got.column("row"))
            assert np.array_equal(g, want), (cond.sexpr(), len(g), len(want), np.setdiff1d(g, want)[:5], np.setdiff1d(want, g)[:5])
    finally:
        pb.close()
        bb.close()


@pytest.mark.parametrize("interpret_only", [False, True], ids=["typed-fast-path", "interpreter"])
def test_join_build_filter_decides_which_rows_enter_the_relation(gpu, stream, interpret_only, sbconfig):
    from spark_b200.execution import BroadcastHashJoinExec, FilterExec, LocalTableScanExec
    from spark_b200.expressions import Cast, Literal, col
    sbconfig("expr_interpret_only", 1 if interpret_only else 0)
    nb = 100_003
    t = adversarial_table(nb, seed=43)
    probe = pa.table({"k": np.random.default_rng(1).permutation(nb).astype(np.int64)})
    conds = join_probe_conditions() + [(Cast(col("f64"), "int") > Literal(0)) | col("b"), (col("i32") * col("i32")) < Literal(0)]
    pb, bb = _scan(probe, stream), _scan(t, stream)
    try:
        for cond in conds:
            got = BroadcastHashJoinExec(["k"], ["row"], "inner", "right", LocalTableScanExec(pb),
                                        FilterExec(cond, LocalTableScanExec(bb))).collect(stream)
            g = np.sort(np.asarray(got.column("row")))
            want = np.flatnonzero(O.filter_mask(t, cond.sexpr()))
            assert np.array_equal(g, want), (cond.sexpr(), len(g), len(want))
            assert np.array_equal(np.asarray(got.column("k")), np.asarray(got.column("row")))
    finally:
        pb.close()
        bb.close()


def _prefixed(t, p):
    return t.rename_columns([p + c for c in t.column_names])


@pytest.mark.parametrize("how", ["inner", "left_outer"])
@pytest.mark.parametrize("npr", [50_000, (1 << 20) + 4097])
@pytest.mark.parametrize("relation", ["duplicates", "dense-unique", "sorted-unique"])
def test_join_residual_condition_per_pair(gpu, stream, how, npr, relation):
    """1:1 keys, so every streamed row has one key match and the condition's verdict on that pair is visible: inner keeps the pairs
    for which it is TRUE, left outer NULL-extends the others.  The pair mask and the pair indices are computed by different passes
    (csrc/join.cu sb_join_probe_condition); each output row must pair a streamed row with its own build row."""
    from spark_b200.execution import BroadcastHashJoinExec, LocalTableScanExec
    from spark_b200.expressions import Cast, Literal, col
    rng = np.random.default_rng(npr)
    nb = 60_000                                  # dense-unique: a permutation of 0..nb-1, range nb <= 8 * nb -> row_of
    if relation == "sorted-unique":
        # csrc/join.cu sb_join_build: unique keys whose range is <= 8 * rows become the direct-address table (row_of) even when
        # ascending; ascending keys over a wider range that is still <= 2^23 (an exact bitmap) take the sorted mode (bitmap + rank)
        keys = np.arange(nb, dtype=np.int64) * 40 + 17
        assert 8 * nb < keys[-1] - keys[0] <= 1 << 23
    else:
        keys = rng.permutation(nb).astype(np.int64)
    probed = nb
    if relation == "duplicates":                 # duplicate keys nobody probes: the dense attempt fails, the relation takes a slot table
        probed = nb - 100
        keys[probed:] = -1 - np.arange(100) % 10
    B = _prefixed(adversarial_table(nb, seed=5), "b_").append_column("k2", pa.array(keys))
    S = _prefixed(adversarial_table(npr, seed=6), "s_")
    idx = rng.integers(0, probed, npr)
    S = S.append_column("k", pa.array(keys[idx]))
    joined = pa.table({**{c: S.column(c) for c in S.column_names}, **{c: B.column(c).take(pa.array(idx)) for c in B.column_names}})
    conds = [((col("s_i32") + col("b_i32")) > Literal(0)) | (Cast(col("s_f64"), "long") < col("b_i64")),
             ((col("s_f64") * col("b_f64")) >= Literal(0.0)) & ~(Cast(col("b_f32"), "int").eq(col("s_i32") - col("b_i8")))]
    sb, bb = _scan(S, stream), _scan(B, stream)
    try:
        for cond in conds:
            got = BroadcastHashJoinExec(["k"], ["k2"], how, "right", LocalTableScanExec(sb), LocalTableScanExec(bb), condition=cond).collect(stream)
            mask = O.filter_mask(joined, cond.sexpr())
            order = np.argsort(np.asarray(got.column("s_row")), kind="stable")
            s_row = np.asarray(got.column("s_row"))[order]
            b_row, b_valid = _host(got.column("b_row"))
            b_row, b_valid = b_row[order], b_valid[order]
            if how == "inner":
                assert np.array_equal(s_row, np.flatnonzero(mask)), (cond.sexpr(), len(s_row), int(mask.sum()))
                assert b_valid.all()
            else:
                assert np.array_equal(s_row, np.arange(npr)), "left outer keeps every streamed row once"
                assert np.array_equal(b_valid, mask), cond.sexpr()
            assert np.array_equal(b_row[b_valid], idx[s_row[b_valid]]), "a pair joined the wrong build row"
    finally:
        sb.close()
        bb.close()


# ---- aggregate ----------------------------------------------------------------------------------------------------------------
def _agg_products():
    from spark_b200.expressions import Literal, col
    return [col("f64"),                                                                            # 1 factor, col
            Literal(1.0) - col("g64"),                                                             # lit - col
            col("f64") * (col("g64") + Literal(0.1)),                                              # col * (col + lit)
            (col("f64") - Literal(0.3)) * (Literal(3.0) + col("g64")) * (Literal(1.0) - col("h64")),  # 3 factors, all modes
            col("f64") * col("g64") * col("h64") * (Literal(1.0) - col("f64"))]                   # 4 factors: materialised


def _agg_conditions(rtc):
    from spark_b200.expressions import Literal, col
    c = [(col("f32") < Literal(NAN)) & (col("i32") >= Literal(-1)) & (col("dt") <= Literal(2)) & col("g64").is_not_null()]
    if not rtc:       # each condition shape is one more NVRTC compile: the specialised runs keep one
        c += [(col("f64") > Literal(-0.0)) & col("b").eq(Literal(True)) & (col("i64") > Literal(I64_MIN)) & (col("ts") < Literal(I64_MAX)),
              (col("i8") < Literal(0)) | (col("f64") >= Literal(NAN))]
    return c


def _order_key(v):
    """The order MIN / MAX use on doubles here: NaN largest, -0.0 < 0.0 (DESIGN §2: the reference keeps whichever arrived first)."""
    v = np.where(np.isnan(v), np.nan, v)
    b = v.view(np.int64)
    return np.where(b < 0, b ^ np.int64(0x7FFFFFFFFFFFFFFF), b)


@pytest.mark.parametrize("env", [{"agg_rtc": 0}, {"agg_rtc_min_rows": 0}], ids=["generic", "rtc"])
def test_aggregate_fused_filter_and_products_per_row(gpu, stream, env, sbconfig):
    """GROUP BY row: every row is its own group, so COUNT(*) shows the fused filter's verdict and SUM(product) the product of that
    row as Spark sums it, add(coalesce(sum, 0), x) (Sum.scala:136-139): a lone -0.0 sums to +0.0, bit for bit."""
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Count, Sum
    for k, v in env.items():
        sbconfig(k, v)
    n = 100_003
    t = adversarial_table(n, seed=77)
    prods = _agg_products()
    aggs = [(Count(), "n")] + [(Sum(p), "s%d" % i) for i, p in enumerate(prods)]
    batch = _scan(t, stream)
    try:
        for cond in _agg_conditions("agg_rtc_min_rows" in env):
            got = HashAggregateExec(["row"], aggs, LocalTableScanExec(batch), condition=cond).collect(stream)
            order = np.argsort(np.asarray(got.column("row")))
            rows = np.flatnonzero(O.filter_mask(t, cond.sexpr()))
            assert np.array_equal(np.asarray(got.column("row"))[order], rows), cond.sexpr()
            assert np.all(np.asarray(got.column("n")) == 1)
            sub = t.take(pa.array(rows))
            for i, p in enumerate(prods):
                x, xv = O.eval_expr(p.sexpr(), sub)
                with np.errstate(invalid="ignore"):                 # NaN products stay NaN
                    want = np.where(xv, 0.0 + x.astype(np.float64), 0.0)
                assert_bits(got.column("s%d" % i).take(pa.array(order)), (want, xv), ("sum", p.sexpr(), cond.sexpr()))
    finally:
        batch.close()


@pytest.mark.parametrize("env", [{"agg_rtc": 0, "agg_tier": 1}, {"agg_rtc": 0, "agg_tier": 2},
                                 {"agg_rtc_min_rows": 0, "agg_tier": 1}, {"agg_rtc_min_rows": 0, "agg_tier": 2}],
                         ids=["generic-dict", "generic-smem", "rtc-dict", "rtc-smem"])
def test_aggregate_min_max_of_products_per_group(gpu, stream, env, sbconfig):
    """A few groups: MIN / MAX of fused products do not depend on the order rows arrive in, so they compare bit for bit."""
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Max, Min
    for k, v in env.items():
        sbconfig(k, v)
    n = 100_003
    t = adversarial_table(n, seed=78)
    prods = _agg_products()[1:]
    aggs = [(f(p), "%s%d" % (f.__name__, i)) for i, p in enumerate(prods) for f in (Min, Max)]
    cond = _agg_conditions(True)[0]
    batch = _scan(t, stream)
    try:
        got = HashAggregateExec(["g"], aggs, LocalTableScanExec(batch), condition=cond).collect(stream)
    finally:
        batch.close()
    order = np.argsort(np.asarray(got.column("g")))
    assert np.array_equal(np.asarray(got.column("g"))[order], np.arange(7))
    sub = O.filter_table(t, cond.sexpr())
    g = np.asarray(sub.column("g"))
    for i, p in enumerate(prods):
        x, xv = O.eval_expr(p.sexpr(), sub)
        key = _order_key(x.astype(np.float64))
        for f in (Min, Max):
            want, wvalid = np.zeros(7), np.zeros(7, bool)
            for grp in range(7):
                m = np.flatnonzero((g == grp) & xv)
                if len(m):
                    j = m[np.argmin(key[m])] if f is Min else m[np.argmax(key[m])]
                    want[grp], wvalid[grp] = x[j], True
            assert_bits(got.column("%s%d" % (f.__name__, i)).take(pa.array(order)), (want, wvalid), (f.__name__, p.sexpr()))


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _refusal_table(n=64):
    import decimal
    rng = np.random.default_rng(9)
    cols = {"k": np.arange(n, dtype=np.int64),
            "price": pa.array([decimal.Decimal(int(v)) / 100 for v in rng.integers(0, 1000, n)], pa.decimal128(12, 2)),
            "s": pa.array(["s%d" % i if i % 5 else None for i in range(n)]), "f": rng.standard_normal(n),
            "i": rng.integers(-5, 5, n).astype(np.int32), "l": rng.integers(-5, 5, n)}
    for c in range(13):
        cols["c%d" % c] = rng.integers(0, 3, n).astype(np.int32)
    return pa.table(cols)


def _bad_programs():
    """name -> (predicate form, value form, expected error code)."""
    from spark_b200.expressions import Cast, Literal, col
    gt0 = lambda vt: [_lit(vt, 0), ("GT", 1, vt, None)]                         # noqa: E731
    cast_arg = [("COL", 4, "f", None), ("CAST_I64", 3, 0, None)]                 # CAST(double AS BIGINT) with arg = 0
    add_mix = [("COL", 2, "i", None), ("COL", 3, "l", None), ("ADD", 3, 0, None)]
    too_deep = [_lit(2, 1)] * 13 + [("ADD", 2, 0, None)] * 12                   # one slot more than EXPR_STACK
    cols13 = [("COL", 2, "c0", None)]
    for c in range(1, 13):
        cols13 += [("COL", 2, "c%d" % c, None), ("ADD", 2, 0, None)]
    return {
        "decimal-compare": (col("price") > Literal(5), Cast(col("price") > Literal(5), "long"), 5),
        "decimal-arithmetic": ((col("price") * Literal(2)) > Literal(5), col("price") * Literal(2), 5),
        "isnull-string": (col("s").is_null(), Cast(col("s").is_null(), "long"), 5),
        "cast-arg-not-operand-class": (Raw(cast_arg + gt0(3)), Raw(cast_arg, vt=3), 2),
        "add-mismatched-operands": (Raw(add_mix + gt0(3)), Raw(add_mix, vt=3), 2),
        "stack-too-deep": (Raw(too_deep + gt0(2)), Raw(too_deep, vt=2), 2),
        "13-distinct-columns": (Raw(cols13 + gt0(2)), Raw(cols13, vt=2), 2),
    }


def _entry_points():
    from spark_b200.execution import (BroadcastHashJoinExec, ExpandExec, FilterExec, HashAggregateExec, LocalTableScanExec,
                                      ProjectExec)
    from spark_b200.expressions import Count, Sum
    S = LocalTableScanExec
    return {
        "filter-fast-path": ("pred", lambda e, a, b: FilterExec(e, S(a))),
        "filter-interpreter": ("pred", lambda e, a, b: FilterExec(e, S(a))),
        "project": ("value", lambda e, a, b: ProjectExec([("v", e)], S(a))),
        "aggregate-condition": ("pred", lambda e, a, b: HashAggregateExec(["k"], [(Count(), "n")], S(a), condition=e)),
        "aggregate-input": ("value", lambda e, a, b: HashAggregateExec(["k"], [(Sum(e), "s")], S(a))),
        "join-build-filter": ("pred", lambda e, a, b: BroadcastHashJoinExec(["k"], ["k"], "inner", "right", S(a), FilterExec(e, S(b)))),
        "join-probe-filter": ("pred", lambda e, a, b: BroadcastHashJoinExec(["k"], ["k"], "inner", "right", FilterExec(e, S(a)), S(b))),
        "join-condition": ("pred", lambda e, a, b: BroadcastHashJoinExec(["k"], ["k"], "inner", "right", S(a), S(b), condition=e)),
        "expand": ("value", lambda e, a, b: ExpandExec([[e]], ["v"], S(a))),
    }


@pytest.mark.parametrize("program", ["decimal-compare", "decimal-arithmetic", "isnull-string", "cast-arg-not-operand-class",
                                     "add-mismatched-operands", "stack-too-deep", "13-distinct-columns"])
@pytest.mark.parametrize("entry", ["filter-fast-path", "filter-interpreter", "project", "aggregate-condition", "aggregate-input",
                                   "join-build-filter", "join-probe-filter", "join-condition", "expand"])
def test_every_entry_point_refuses_what_it_cannot_evaluate(gpu, stream, entry, program, sbconfig):
    """Comparisons / arithmetic on DECIMAL columns (unscaled values would ignore the scale) and IS NULL over strings are
    SB_ERR_UNSUPPORTED; programs whose vtypes disagree (what a compiler passing arg = 0 to every CAST emits), that need more stack
    slots or more distinct columns than the kernels hold are SB_ERR_INVALID.  Every operator validates before it evaluates."""
    from spark_b200 import _capi as capi
    sbconfig("expr_interpret_only", 1 if entry == "filter-interpreter" else 0)
    kind, plan = _entry_points()[entry]
    pred, value, code = _bad_programs()[program]
    t = _refusal_table()
    a, b = _scan(t, stream), _scan(t, stream)
    try:
        with pytest.raises(capi.SparkB200Error) as ei:
            plan(pred if kind == "pred" else value, a, b).collect(stream)
        assert ei.value.code == code, str(ei.value)
    finally:
        a.close()
        b.close()


def test_decimal_null_tests_and_bare_references_still_work(gpu, stream):
    from spark_b200.execution import FilterExec, LocalTableScanExec, ProjectExec
    from spark_b200.expressions import col
    t = _refusal_table()
    t = t.set_column(1, "price", pa.array([None if i % 3 == 0 else v for i, v in enumerate(t.column("price").to_pylist())], pa.decimal128(12, 2)))
    cols12 = [("COL", 2, "c0", None)]
    for c in range(1, 12):
        cols12 += [("COL", 2, "c%d" % c, None), ("ADD", 2, 0, None)]
    deep = [_lit(2, 1)] * 12 + [("ADD", 2, 0, None)] * 11
    batch = _scan(t, stream)
    try:
        got = ProjectExec([("k", col("k")), ("price", col("price")), ("nn", col("price").is_not_null()), ("c12", Raw(cols12, vt=2)),
                           ("deep", Raw(deep, vt=2))],
                          FilterExec(col("price").is_not_null(), LocalTableScanExec(batch))).collect(stream)
    finally:
        batch.close()
    keep = [i for i in range(t.num_rows) if i % 3]
    assert got.column("k").to_pylist() == keep
    assert got.column("price").to_pylist() == [t.column("price")[i].as_py() for i in keep]
    assert all(got.column("nn").to_pylist())
    assert got.column("c12").to_pylist() == [sum(t.column("c%d" % c)[i].as_py() for c in range(12)) for i in keep]
    assert got.column("deep").to_pylist() == [12] * len(keep)
