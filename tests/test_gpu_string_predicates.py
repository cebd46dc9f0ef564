"""String tests against literals on the GPU (SB_OP_STR_*), bit-exact against tests/string_oracle.py.

Every program with a string test runs on the interpreter (csrc/expr.cu eval_row with the matchers of csrc/strpred.cuh), whichever
operator evaluates it.  The data holds empty strings, NULLs, strings equal to and prefixes of the literals, literals longer than
the row, 2-, 3- and 4-byte code points, `%`, `_` and `\\` in the data, 0x00 / 0xFF bytes (in the column the byte-level tests read)
and 70 KB strings among short ones."""
import numpy as np
import pyarrow as pa
import pytest

import string_oracle as SO

pytestmark = pytest.mark.gpu

WORDS = ["", "BUILDING", "BUILDIN", "BUILDINGS", "AUTOMOBILE", "MACHINERY", "ASIA", "AS", "a", "ab", "abc", "€", "a€a", "€€",
         "😀😇🥑", "😀", "日本語", "ß", "100%", "a_b", "a\\b", "%", "_", "\\", "\\\\", "a\nb", "\n", "PROMO BRUSHED BRASS",
         "STANDARD POLISHED BRASS", "PROMO ANODIZED TIN", "ECONOMY BRASS ", "forest green lime", "greenish", "GREEN",
         "carefully special requests", "special requests", "requests special", "x special y requests z", "PROMO%", "é"]
BYTES = [b"\x00", b"\xff", b"a\x00b", b"\xffa", b"BUILDING\x00", b"\x00\x00", b"a\xff"]
LONG = 70_000


def string_table(n, seed):
    """Columns: s (valid UTF-8, NULLs, every ~5000th row a LONG string), b (bytes incl. 0x00 / 0xFF, NULLs), x (int32), row."""
    rng = np.random.default_rng(seed)
    words = [w.encode() for w in WORDS]
    pick = rng.integers(0, len(words), n)
    s = [words[i] for i in pick]
    rnd = rng.random(n)
    for r in np.flatnonzero(rnd < 0.2):            # random concatenations of two words
        s[r] = words[pick[r]] + words[(pick[r] * 7 + 3) % len(words)]
    for r in range(17, n, 5000):
        s[r] = ("special " + "é" * (LONG // 2) + " requests").encode()
    s_null = rng.random(n) < 0.1
    bpool = words + BYTES
    b = [bpool[i] for i in rng.integers(0, len(bpool), n)]
    b_null = rng.random(n) < 0.1
    return pa.table({"s": _binary_string(s, s_null), "b": _binary_string(b, b_null),
                     "x": rng.integers(-3, 4, n).astype(np.int32), "row": np.arange(n, dtype=np.int64)})


def _binary_string(vals, nulls, first_offset=0):
    """An Arrow string column built from raw bytes (no UTF-8 validation), offsets starting at `first_offset`."""
    n = len(vals)
    offs = np.cumsum([first_offset] + [0 if nl else len(v) for v, nl in zip(vals, nulls)]).astype(np.int32)
    data = b"\x07" * first_offset + b"".join(v for v, nl in zip(vals, nulls) if not nl)
    valid = pa.py_buffer(np.packbits(~np.asarray(nulls, bool), bitorder="little").tobytes()) if n else None
    return pa.Array.from_buffers(pa.string(), n, [valid, pa.py_buffer(offs.tobytes()), pa.py_buffer(data)], null_count=int(np.sum(nulls)))


def byte_tests(c):
    from spark_b200.expressions import Contains, EndsWith, EqualTo, GreaterThan, In, LessThan, LessThanOrEqual, Literal, StartsWith, col
    s = col(c)
    lits = ["BUILDING", "", "BUILDINGS", "€", "a", "\\", b"\x00", b"\xff", "😀😇🥑x"]
    out = []
    for v in lits:
        out += [EqualTo(s, Literal(v)), StartsWith(s, v), EndsWith(s, v), Contains(s, v)]
    for v in ("BUILDING", "a", "", b"\xff", "€"):
        out += [LessThan(s, Literal(v)), LessThanOrEqual(Literal(v), s), GreaterThan(s, Literal(v)), s >= Literal(v), s.ne(v)]
    out += [In(s, ["AUTOMOBILE", "BUILDING", "MACHINERY", "HOUSEHOLD", "FURNITURE", "BUILDING", b"\xff"]), In(s, ["a", None]),
            In(s, []), In(s, [None]), ~In(s, ["ab", None]), ~In(s, ["ab", "abc"])]
    return out


def like_tests():
    from spark_b200.expressions import Like, col
    s = col("s")
    pats = ["%BRASS", "PROMO%", "%green%", "%special%requests%", "BUILDING", "", "%", "_", "__", "___", "a_b", "a\\_b", "a\\%", "%\\%",
            "\\\\", "%\\\\%", "_€_", "😀_🥑", "%🥑", "😀%", "a%b", "%a%b%", "%é%é%", "_%_", "%_%_%", "a\nb", "%\n%", "a_%b", "%%", "PROMO_%"]
    out = [Like(s, p) for p in pats]
    out += [~Like(s, "%special%requests%"), Like(s, "a!%", escape="!"), Like(s, "!!%", escape="!"), Like(s, "%€%", escape="€")]
    return out


def all_predicates():
    from spark_b200.expressions import Literal, OctetLength, StartsWith, col
    p = byte_tests("s") + byte_tests("b") + like_tests()
    p += [(col("x") > Literal(0)) & col("s").eq("BUILDING"), StartsWith(col("s"), "PROMO") & (col("x") <= Literal(1)) & ~StartsWith(col("b"), "a"),
          (OctetLength(col("s")) > Literal(3)) | col("b").eq(b"\x00"), col("s").eq("ASIA") | (col("x") > Literal(2))]
    return p


def _scan(t, stream):
    from spark_b200.columnar import ColumnarBatch
    return ColumnarBatch.from_arrow(t, stream)


def _filter_rows(batch, cond, stream):
    from spark_b200.execution import FilterExec, LocalTableScanExec, ProjectExec
    return np.asarray(ProjectExec(["row"], FilterExec(cond, LocalTableScanExec(batch))).collect(stream).column("row"))


_TABLES, _MASKS = {}, {}


def _table(n):
    if n not in _TABLES:
        _TABLES[n] = string_table(n, seed=n)
    return _TABLES[n]


def _oracle_rows(n, cond):
    key = (n, repr(cond.sexpr()))
    if key not in _MASKS:
        _MASKS[key] = np.flatnonzero(SO.filter_mask(_table(n), cond.sexpr()))
    return _MASKS[key]


@pytest.mark.parametrize("n", [0, 1, 255, 257, 2_000_003])
def test_every_string_test_filters_like_the_oracle(gpu, stream, n):
    """Every test on the small tables (one and two 256-thread blocks); every tenth one and the mixed conjunctions at 2 M rows (the
    oracle is Python)."""
    t = _table(n)
    preds = all_predicates()
    if n > 100_000:
        preds = preds[::10] + preds[-4:]
    batch = _scan(t, stream)
    try:
        for cond in preds:
            g = _filter_rows(batch, cond, stream)
            w = _oracle_rows(n, cond)
            assert np.array_equal(g, w), (cond.sexpr(), len(g), len(w), np.setdiff1d(g, w)[:5], np.setdiff1d(w, g)[:5])
    finally:
        batch.close()


def test_offsets_that_do_not_start_at_zero(gpu, stream):
    """Arrow allows offsets[0] > 0: a string's bytes are wherever its offsets point."""
    from spark_b200.expressions import Like, col
    rng = np.random.default_rng(5)
    n = 5000
    vals = [WORDS[i].encode() for i in rng.integers(0, len(WORDS), n)]
    nulls = rng.random(n) < 0.1
    for first in (1, 13, 16):
        t = pa.table({"s": _binary_string(vals, nulls, first_offset=first), "row": np.arange(n, dtype=np.int64)})
        batch = _scan(t, stream)
        try:
            for cond in (col("s").eq("BUILDING"), Like(col("s"), "%a%"), col("s") < "B"):
                assert np.array_equal(_filter_rows(batch, cond, stream), np.flatnonzero(SO.filter_mask(t, cond.sexpr()))), (first, cond.sexpr())
        finally:
            batch.close()


@pytest.mark.parametrize("n", [1025, 100_003])
def test_projections_of_string_tests(gpu, stream, n):
    """ProjectExec of BOOL string tests and octet_length, over every row and below a filter, NULLs included."""
    from spark_b200.execution import FilterExec, LocalTableScanExec, ProjectExec
    from spark_b200.expressions import Cast, In, Like, Literal, OctetLength, col
    t = string_table(n, seed=3)
    exprs = [OctetLength(col("s")), OctetLength(col("b")), Like(col("s"), "%é%"), In(col("s"), ["a", None]), ~In(col("b"), ["ab", None]),
             col("s").eq("BUILDING") | (col("x") > Literal(0)), Cast(OctetLength(col("s")), "long") * Literal(2), col("s") >= "a",
             OctetLength(col("s")) + OctetLength(col("b"))]
    batch = _scan(t, stream)
    try:
        for filtered in (False, True):
            cond = Like(col("s"), "%a%")
            src = t.take(pa.array(np.flatnonzero(SO.filter_mask(t, cond.sexpr())))) if filtered else t
            child = FilterExec(cond, LocalTableScanExec(batch)) if filtered else LocalTableScanExec(batch)
            got = ProjectExec([("p%d" % i, e) for i, e in enumerate(exprs)], child).collect(stream)
            assert got.num_rows == src.num_rows
            for i, e in enumerate(exprs):
                v, valid = SO.eval_expr(e.sexpr(), src)
                gc = got.column("p%d" % i)
                assert gc.is_valid().to_pylist() == valid.tolist(), e.sexpr()
                gv = np.array([0 if x is None else int(x) for x in gc.to_pylist()], np.int64)
                assert np.array_equal(gv[valid], v[valid].astype(np.int64)), e.sexpr()
    finally:
        batch.close()


def test_ill_formed_utf8_deviation(gpu, stream):
    """DESIGN §2: a code point starts at a string's first byte and at every later byte that is not 10xxxxxx.  Spark decodes first,
    so b'a\\x80' is two characters ('a', U+FFFD) to it and one code point here; b'\\x80a' is two for both."""
    from spark_b200.execution import LocalTableScanExec, ProjectExec
    from spark_b200.expressions import Like, col
    t = pa.table({"s": _binary_string([b"a\x80", b"\xff\xfe", b"\x80a"], [False] * 3)})
    batch = _scan(t, stream)
    try:
        got = ProjectExec([("two", Like(col("s"), "__")), ("one", Like(col("s"), "_"))], LocalTableScanExec(batch)).collect(stream)
    finally:
        batch.close()
    assert got.column("two").to_pylist() == [False, True, True]
    assert got.column("one").to_pylist() == [True, False, False]


# ---- every entry point that takes a program ----------------------------------------------------------------------------------
def test_string_tests_in_aggregate_join_and_expand(gpu, stream):
    from spark_b200.execution import BroadcastHashJoinExec, ExpandExec, FilterExec, HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Count, In, Like, Literal, OctetLength, Sum, col
    n = 200_003
    t = string_table(n, seed=11).append_column("g", pa.array((np.arange(n) % 5).astype(np.int32)))
    conds = [Like(col("s"), "%BRASS"), col("s").eq("BUILDING") & (col("x") >= Literal(0)), ~Like(col("s"), "%special%requests%"),
             In(col("b"), ["a", "ab", None]) | (OctetLength(col("s")) > Literal(20))]
    S = LocalTableScanExec
    batch = _scan(t, stream)
    keys = pa.table({"k": np.arange(n, dtype=np.int64)})
    kb = _scan(keys, stream)
    try:
        for cond in conds:
            mask = SO.filter_mask(t, cond.sexpr())
            rows = np.flatnonzero(mask)
            got = HashAggregateExec(["g"], [(Count(), "n"), (Sum(OctetLength(col("s"))), "len")], S(batch), condition=cond).collect(stream)
            order = np.argsort(np.asarray(got.column("g")))
            g = np.asarray(t.column("g"))[rows]
            lens, lvalid = SO.eval_expr(("octet_length", ("col", "s")), t)
            assert np.asarray(got.column("n"))[order].tolist() == [int(np.sum(g == k)) for k in np.unique(g)], cond.sexpr()
            want_len = [int(np.sum(lens[rows][(g == k) & lvalid[rows]])) for k in np.unique(g)]
            assert np.asarray(got.column("len"))[order].tolist() == want_len, cond.sexpr()
            # join: build filter, probe filter, residual condition over the streamed side's string column
            j = BroadcastHashJoinExec(["k"], ["row"], "inner", "right", S(kb), FilterExec(cond, S(batch))).collect(stream)
            assert np.array_equal(np.sort(np.asarray(j.column("row"))), rows), ("build", cond.sexpr())
            j = BroadcastHashJoinExec(["row"], ["k"], "left_semi", "right", FilterExec(cond, S(batch)), S(kb)).collect(stream)
            assert np.array_equal(np.asarray(j.column("row")), rows), ("probe", cond.sexpr())
            j = BroadcastHashJoinExec(["row"], ["k"], "inner", "right", S(batch), S(kb), condition=cond).collect(stream)
            assert np.array_equal(np.sort(np.asarray(j.column("row"))), rows), ("condition", cond.sexpr())
        got = ExpandExec([[Like(col("s"), "%a%"), OctetLength(col("s"))], [col("s").eq("BUILDING"), OctetLength(col("b"))]], ["t", "len"],
                         S(batch)).collect(stream)
        want_t = [SO.eval_expr(e, t) for e in (("like", ("col", "s"), "%a%", "\\"), ("str_cmp", "eq", ("col", "s"), ("lit", "BUILDING", str)))]
        want_l = [SO.eval_expr(("octet_length", ("col", c)), t) for c in ("s", "b")]
        for l in range(2):
            gt, gl = got.column("t").to_pylist()[l::2], got.column("len").to_pylist()[l::2]
            assert gt == [bool(v) if ok else None for v, ok in zip(*want_t[l])]
            assert gl == [int(v) if ok else None for v, ok in zip(*want_l[l])]
    finally:
        batch.close()
        kb.close()


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _bad_string_programs():
    """name -> raw nodes (op, vtype, arg, arg2, lit) and pool bytes; every one is SB_ERR_INVALID."""
    import struct
    rec = struct.pack("=I", 2) + struct.pack("=I", 1) + b"a" + struct.pack("=I", 5) + b"b"       # second record overruns
    return {
        "slice-outside-pool": ([("STR_EQ", 1, "s", 0, 4 << 32 | 4)], b"abcdef"),
        "non-string-column": ([("STR_STARTS_WITH", 1, "k", 0, 1)], b"a"),
        "escape-at-the-end": ([("STR_LIKE", 1, "s", 92, 2)], b"a\\"),
        "escape-in-the-middle": ([("STR_LIKE", 1, "s", 92, 2)], b"\\a"),
        "bad-in-records": ([("STR_IN", 1, "s", 0, len(rec))], rec),
        "in-arg2-not-0-or-1": ([("STR_IN", 1, "s", 2, 4)], struct.pack("=I", 0)),
        "octet-length-not-i32": ([("STR_OCTET_LENGTH", 1, "s", 0, 0)], b""),
    }


class _RawString:
    """A hand-built program with its own pool (bypasses the Python nodes' checks)."""

    def __init__(self, nodes, pool):
        self.nodes, self.pool = nodes, pool

    def vtype(self, schema):
        return 1

    def emit(self, schema, out):
        from spark_b200.expressions import _node
        out.pool += self.pool
        for op, vt, arg, arg2, lit in self.nodes:
            out.append(_node(op, vt, schema.index(arg), lit_i=lit, arg2=arg2))

    def references(self):
        return {a for _, _, a, _, _ in self.nodes}

    def sexpr(self):
        return None


@pytest.mark.parametrize("program", sorted(_bad_string_programs()))
@pytest.mark.parametrize("entry", ["filter", "project", "aggregate-condition", "aggregate-input",
                                   "join-build-filter", "join-probe-filter", "join-condition", "expand"])
def test_every_entry_point_refuses_malformed_string_tests(gpu, stream, entry, program):
    from spark_b200 import _capi as capi
    from spark_b200.execution import (BroadcastHashJoinExec, ExpandExec, FilterExec, HashAggregateExec, LocalTableScanExec, ProjectExec)
    from spark_b200.expressions import Count, Expression, Sum

    class Raw(_RawString, Expression):
        pass
    nodes, pool = _bad_string_programs()[program]
    e = Raw(nodes, pool)
    S = LocalTableScanExec
    plans = {
        "filter": lambda a, b: FilterExec(e, S(a)),
        "project": lambda a, b: ProjectExec([("v", e)], S(a)),
        "aggregate-condition": lambda a, b: HashAggregateExec(["k"], [(Count(), "n")], S(a), condition=e),
        "aggregate-input": lambda a, b: HashAggregateExec(["k"], [(Sum(e), "s")], S(a)),
        "join-build-filter": lambda a, b: BroadcastHashJoinExec(["k"], ["k"], "inner", "right", S(a), FilterExec(e, S(b))),
        "join-probe-filter": lambda a, b: BroadcastHashJoinExec(["k"], ["k"], "inner", "right", FilterExec(e, S(a)), S(b)),
        "join-condition": lambda a, b: BroadcastHashJoinExec(["k"], ["k"], "inner", "right", S(a), S(b), condition=e),
        "expand": lambda a, b: ExpandExec([[e]], ["v"], S(a)),
    }
    t = pa.table({"k": np.arange(64, dtype=np.int64), "s": pa.array(["s%d" % i if i % 5 else None for i in range(64)])})
    a, b = _scan(t, stream), _scan(t, stream)
    try:
        with pytest.raises(capi.SparkB200Error) as ei:
            plans[entry](a, b).collect(stream)
        assert ei.value.code == 2, str(ei.value)
    finally:
        a.close()
        b.close()


# ---- end to end: Q3 and Q5 over real string columns ---------------------------------------------------------------------------
REGIONS = ["AFRICA", "AMERICA", "ASIA", "EUROPE", "MIDDLE EAST"]      # TPC-H r_name by r_regionkey


def _with_string_filter(plan, column, value):
    """The plan with its FilterExec on `column` = code replaced by `column` = 'value' (the predicate a real plan carries)."""
    from spark_b200.execution import FilterExec
    from spark_b200.expressions import col
    seen, stack, hits = set(), [plan], 0
    while stack:
        p = stack.pop()
        if id(p) in seen:
            continue
        seen.add(id(p))
        if isinstance(p, FilterExec) and p.condition.references() == {column}:
            p.condition = col(column).eq(value)
            hits += 1
        stack += [c for c in getattr(p, "children", ()) if c is not None]
        stack += [getattr(p, a) for a in ("child", "left", "right") if getattr(p, a, None) is not None]
    assert hits == 1, hits
    return plan


def _scan_plan(t, stream):
    from spark_b200.execution import LocalTableScanExec
    return LocalTableScanExec(_scan(t, stream))


def test_q3_and_q5_filter_real_string_columns(gpu, stream):
    """c_mktsegment / r_name as strings (tpch.SEGMENTS[code], TPC-H region names) filtered with = 'BUILDING' / = 'ASIA' give the
    answers of the code-based oracle."""
    from oracle import tpch_oracle as TO
    from spark_b200 import tpch
    from util import assert_tables_equal
    assert tpch.SEGMENTS[tpch.Q3_SEGMENT] == "BUILDING" and REGIONS[tpch.Q5_REGION] == "ASIA"
    sf = 0.05
    customer, orders = tpch.customer_table(sf), tpch.orders_table(sf)
    lineitem = tpch.lineitem_join_table(orders, sf)
    supplier, nation, region = tpch.supplier_table(sf), tpch.nation_table(), tpch.region_table()
    seg = customer.column("c_mktsegment").to_numpy()
    customer_s = customer.set_column(customer.schema.get_field_index("c_mktsegment"), "c_mktsegment", pa.array([tpch.SEGMENTS[c] for c in seg]))
    region_s = region.set_column(region.schema.get_field_index("r_name"), "r_name", pa.array([REGIONS[c] for c in region.column("r_name").to_numpy()]))

    plan = _with_string_filter(tpch.q3_plan(_scan_plan(customer_s, stream), _scan_plan(orders, stream), _scan_plan(lineitem, stream)),
                               "c_mktsegment", "BUILDING")
    got = plan.collect(stream)
    want, all_groups = TO.q3(customer, orders, lineitem, tpch.Q3_SEGMENT, tpch.Q3_DATE)
    assert all_groups.num_rows > 100
    assert got.column("l_orderkey").to_pylist() == want.column("l_orderkey").to_pylist()
    assert_tables_equal(got, want, ordered=True)

    plan = _with_string_filter(tpch.q5_plan(*[_scan_plan(t, stream) for t in (customer_s, orders, lineitem, supplier, nation, region_s)]),
                               "r_name", "ASIA")
    got = plan.collect(stream)
    want = TO.q5(customer, orders, lineitem, supplier, nation, region, tpch.Q5_REGION, tpch.Q5_DATE_LO, tpch.Q5_DATE_HI)
    assert want.num_rows == 5
    assert got.column("n_name").to_pylist() == want.column("n_name").to_pylist()
    assert_tables_equal(got, want, ordered=True)
