"""String-producing functions on the GPU (sb_string_project, csrc/strfunc.cu) and the LENGTH leaf, bit-exact against
tests/string_functions_oracle.py: output bytes, int32 offsets from 0 and validity.  The data holds random UTF-8 of 1-4-byte code
points and emoji, empty strings, NULLs, lone continuation bytes and truncated lead bytes at the end of values."""
import json
import os

import numpy as np
import pyarrow as pa
import pytest

import string_functions_oracle as O

pytestmark = pytest.mark.gpu

INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
CPS = ["a", "Z", " ", "-", "0", "é", "ß", "€", "日", "本", "😀", "🥑", "𝄞"]
ILL = [b"\x80", b"\xbf", b"\xc0", b"\xff", b"\xe4\xb8", b"\xf0\x9f\x98"]


def _binary_string(vals):
    """An Arrow string column from raw bytes / None (no UTF-8 validation)."""
    nulls = [v is None for v in vals]
    offs = np.cumsum([0] + [0 if v is None else len(v) for v in vals]).astype(np.int32)
    data = b"".join(v for v in vals if v is not None)
    valid = pa.py_buffer(np.packbits(~np.asarray(nulls, bool), bitorder="little").tobytes()) if vals else None
    return pa.Array.from_buffers(pa.string(), len(vals), [valid, pa.py_buffer(offs.tobytes()), pa.py_buffer(data)], null_count=sum(nulls))


def random_strings(n, seed, null_p=0.1, ill=True):
    rng = np.random.default_rng(seed)
    cps = [c.encode() for c in CPS]
    lens = rng.integers(0, 12, n)
    out = []
    for i in range(n):
        v = b"".join(cps[k] for k in rng.integers(0, len(cps), lens[i]))
        r = rng.random()
        if ill and r < 0.05:
            v = v + ILL[rng.integers(0, len(ILL))]           # truncated lead byte / stray byte at the end
        elif ill and r < 0.1:
            v = ILL[rng.integers(0, 4)] + v                  # lone continuation byte or a disallowed lead first
        out.append(None if rng.random() < null_p else v)
    return out


def _golden_bytes(x):
    """a golden string: UTF-8 text, {"hex": ...} for raw bytes, or None"""
    if isinstance(x, dict):
        return bytes.fromhex(x["hex"])
    return None if x is None else x.encode()


def _scan(t, stream):
    from spark_b200.columnar import ColumnarBatch
    return ColumnarBatch.from_arrow(t, stream)


def assert_column(arr, want, what=""):
    """offsets from 0, bytes and validity exactly as the oracle's values"""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    assert arr.type == pa.string() and len(arr) == len(want), what
    valid, offs, data = arr.buffers()
    offs = np.frombuffer(offs, np.int32, len(want) + 1, arr.offset * 4) if len(want) else np.zeros(1, np.int32)
    wl = np.array([0 if v is None else len(v) for v in want], np.int64)
    assert offs[0] == 0 and np.array_equal(np.diff(offs.astype(np.int64)), wl), what
    got = bytes(data)[:int(offs[-1])] if data is not None else b""
    assert got == b"".join(v for v in want if v is not None), what
    assert arr.is_null().to_pylist() == [v is None for v in want], what


def project(batch, exprs, stream):
    from spark_b200.execution import LocalTableScanExec, ProjectExec
    return ProjectExec([("o%d" % i, e) for i, e in enumerate(exprs)], LocalTableScanExec(batch)).collect(stream)


def oracle(e, t):
    cols = {n: t.column(n).cast(pa.binary()).to_pylist() if t.schema.field(n).type == pa.string() else t.column(n).to_pylist()
            for n in t.column_names}
    return [O.evaluate(e, {k: v[r] for k, v in cols.items()}) for r in range(t.num_rows)]


def edge_exprs():
    from spark_b200.expressions import (Concat, ConcatWs, StringLPad, StringRPad, StringTrim, StringTrimLeft, StringTrimRight, Substring,
                                        col)
    s = col("s")
    out = [Substring(s, p, l) for p in (0, 1, -1, 2, -3, 7, 100, INT_MAX, INT_MIN) for l in (0, 1, -1, 2, 5, INT_MAX, INT_MIN)]
    out += [Substring(s, 3), Substring(s, -2)]
    out += [Concat(s, "-", col("t")), Concat(s), Concat(s, None), ConcatWs("·", s, col("t"), "x"), ConcatWs("", s, col("t")), ConcatWs(None, s)]
    out += [StringTrim(s), StringTrimLeft(s), StringTrimRight(s), StringTrim(s, "a 😀"), StringTrimLeft(s, "€é\x80"), StringTrimRight(s, "日\xbf"),
            StringTrim(s, ""), StringTrim(s, None), StringTrim(s, b"\xc3\xa9")]
    out += [StringLPad(s, n, p) for n in (0, -1, INT_MIN, 1, 5, 20) for p in ("0", "", "ab€", "😀")]
    out += [StringRPad(s, n, p) for n in (0, 3, 17) for p in ("-", "", "é日")]
    out += [StringLPad(s, 5, None), StringRPad(s, None, "x"), Substring(s, None, 3)]
    # nesting
    out += [Concat(Substring(s, 1, 2), "-", StringTrim(col("t"))), StringLPad(Concat(s, col("t")), 9, "*"),
            Substring(StringRPad(s, 30, "ab"), -4, 3), StringTrim(Concat(" ", s, " ")), ConcatWs(",", Substring(s, 2), None, StringLPad(col("t"), 3, "0")),
            Substring(Concat(col("t"), s), 3, 4), StringTrimRight(Concat(s, "\xe4"), "\xe4")]
    return out


def test_goldens(gpu, stream):
    from spark_b200.expressions import (Concat, ConcatWs, Length, StringLPad, StringRPad, StringTrim, StringTrimLeft, StringTrimRight, Substring,
                                        col)
    with open(os.path.join(os.path.dirname(__file__), "golden", "string_functions.json"), encoding="utf-8") as f:
        vectors = json.load(f)["vectors"]
    fns = {"trim": StringTrim, "ltrim": StringTrimLeft, "rtrim": StringTrimRight}
    for v in vectors:
        a, fn = v["args"], v["fn"]
        want = v["expect"]
        if fn in ("concat", "concat_ws"):
            strs = a if fn == "concat" else a[1:]
            t = pa.table({"c%d" % i: _binary_string([_golden_bytes(x)]) for i, x in enumerate(strs)} or {"z": [0]})
            cs = [col("c%d" % i) for i in range(len(strs))]
            e = Concat(*cs) if fn == "concat" else ConcatWs(a[0], *cs)
        else:
            t = pa.table({"s": _binary_string([_golden_bytes(a[0])])})
            if fn == "substring":
                e = Substring(col("s"), a[1], a[2])
            elif fn in fns:
                e = fns[fn](col("s")) if len(a) == 1 else fns[fn](col("s"), _golden_bytes(a[1]))
            elif fn == "lpad":
                e = StringLPad(col("s"), a[1], a[2])
            elif fn == "rpad":
                e = StringRPad(col("s"), a[1], a[2])
            else:
                e = Length(col("s"))
        b = _scan(t, stream)
        try:
            got = project(b, [e], stream).column("o0")
        finally:
            b.close()
        if fn == "length":
            assert got.to_pylist() == [want], v
        else:
            assert_column(got, [None if want is None else want.encode()], v)


def test_edges_random_and_ill_formed(gpu, stream):
    n = 20_011
    t = pa.table({"s": _binary_string(random_strings(n, 1)), "t": _binary_string(random_strings(n, 2, null_p=0.3))})
    b = _scan(t, stream)
    try:
        exprs = edge_exprs()
        for k in range(0, len(exprs), 16):
            chunk = exprs[k:k + 16]
            got = project(b, chunk, stream)
            for i, e in enumerate(chunk):
                assert_column(got.column("o%d" % i), oracle(e, t), e.sexpr())
    finally:
        b.close()


def test_row_counts_and_all_null(gpu, stream):
    from spark_b200.expressions import Concat, ConcatWs, StringLPad, Substring, col
    exprs = [Substring(col("s"), 2, 3), Concat(col("s"), "|", col("s")), ConcatWs("-", col("s"), col("s")), StringLPad(col("s"), 4, "ab")]
    for vals in ([], [b"\xf0\x9f\x98\x80x"], [None, None, None], [b"", b"", None]):
        t = pa.table({"s": _binary_string(vals)})
        b = _scan(t, stream)
        try:
            got = project(b, exprs, stream)
            for i, e in enumerate(exprs):
                assert_column(got.column("o%d" % i), oracle(e, t), (vals, e.sexpr()))
        finally:
            b.close()
    # 2^20 + 3 rows, with a value longer than the per-thread copy threshold in every warp
    n = (1 << 20) + 3
    vals = random_strings(n, 5)
    for r in range(0, n, 29):
        vals[r] = "日本語😀".encode() * 40
    t = pa.table({"s": _binary_string(vals)})
    b = _scan(t, stream)
    try:
        exprs = [Substring(col("s"), 1, 2), Concat(col("s"), "-", col("s")), StringLPad(col("s"), 70, "0é")]
        got = project(b, exprs, stream)
        for i, e in enumerate(exprs):
            assert_column(got.column("o%d" % i), oracle(e, t), e.sexpr())
    finally:
        b.close()


def test_range_cap_and_refusals(gpu, stream):
    from spark_b200 import _capi as capi
    from spark_b200.expressions import Concat, ConcatWs, StringLPad, col
    t = pa.table({"s": _binary_string([b"ab", None, b"\xe4"])})
    b = _scan(t, stream)
    try:
        at_cap = [Concat(*([col("s")] * 16)), ConcatWs("-", *([col("s")] * 8)), StringLPad(Concat(*([col("s")] * 15)), 40, "x")]
        got = project(b, at_cap, stream)
        for i, e in enumerate(at_cap):
            assert_column(got.column("o%d" % i), oracle(e, t), e.sexpr())
        for e in (Concat(*([col("s")] * 17)), ConcatWs("-", *([col("s")] * 9)), StringLPad(Concat(*([col("s")] * 16)), 40, "x")):
            with pytest.raises(capi.SparkB200Error) as ei:
                project(b, [e], stream)
            assert ei.value.code == 5 and "byte ranges" in str(ei.value)
    finally:
        b.close()
    # an output just over 2^31 - 1 bytes is refused before anything is written
    t = pa.table({"s": _binary_string([b"a", b"b", b"c"])})
    b = _scan(t, stream)
    try:
        with pytest.raises(capi.SparkB200Error) as ei:
            project(b, [StringLPad(col("s"), (1 << 31) // 3 + 1, "z")], stream)
        assert ei.value.code == 5 and "output 0" in str(ei.value)
        got = project(b, [StringLPad(col("s"), 1000, "z")], stream)
        assert got.column("o0").to_pylist() == ["z" * 999 + c for c in "abc"]
    finally:
        b.close()
    # one row over 2^31 - 1 bytes, and rows of 2^36 bytes that would wrap an int64 sum of exact lengths, are refused the same way
    t = pa.table({"s": _binary_string([b"a"])})
    b = _scan(t, stream)
    try:
        with pytest.raises(capi.SparkB200Error) as ei:
            project(b, [StringLPad(col("s"), INT_MAX, "😀")], stream)
        assert ei.value.code == 5 and "output 0" in str(ei.value)
    finally:
        b.close()
    n = 1 << 20
    t = pa.table({"s": _binary_string([b""] * n)})
    b = _scan(t, stream)
    try:
        with pytest.raises(capi.SparkB200Error) as ei:
            project(b, [Concat(*[StringLPad(col("s"), INT_MAX, "😀")] * 8)], stream)
        assert ei.value.code == 5 and "output 0" in str(ei.value)
    finally:
        b.close()
    # binary inputs are refused
    bt = pa.table({"s": pa.array([b"ab"], pa.binary())})
    b = _scan(bt, stream)
    try:
        with pytest.raises(capi.SparkB200Error) as ei:
            project(b, [StringLPad(col("s"), 3, "x")], stream)
        assert ei.value.code == 5
    finally:
        b.close()


def test_length_in_every_entry_point(gpu, stream):
    from spark_b200.execution import (BroadcastHashJoinExec, ExpandExec, FilterExec, HashAggregateExec, LocalTableScanExec, ProjectExec)
    from spark_b200.expressions import Count, Length, Literal, OctetLength, Sum, col
    S = LocalTableScanExec
    n = 50_003
    vals = random_strings(n, 9)
    t = pa.table({"s": _binary_string(vals), "g": (np.arange(n) % 5).astype(np.int32), "row": np.arange(n, dtype=np.int64)})
    lens = [O.length(v) for v in vals]
    b = _scan(t, stream)
    kb = _scan(pa.table({"k": np.arange(n, dtype=np.int64)}), stream)
    try:
        cond = Length(col("s")) > Literal(4)
        rows = [r for r in range(n) if lens[r] is not None and lens[r] > 4]
        got = ProjectExec([("l", Length(col("s"))), ("d", Length(col("s")) - OctetLength(col("s")))], S(b)).collect(stream)
        assert got.column("l").to_pylist() == lens
        assert got.column("d").to_pylist() == [None if v is None else O.length(v) - len(v) for v in vals]
        assert FilterExec(cond, S(b)).collect(stream).column("row").to_pylist() == rows
        agg = HashAggregateExec(["g"], [(Count(), "n"), (Sum(Length(col("s"))), "len")], S(b), condition=cond).collect(stream)
        want = {}
        for r in rows:
            k = r % 5
            c, s_ = want.get(k, (0, 0))
            want[k] = (c + 1, s_ + lens[r])
        assert {g: (c, s_) for g, c, s_ in zip(*[agg.column(x).to_pylist() for x in ("g", "n", "len")])} == want
        j = BroadcastHashJoinExec(["row"], ["k"], "inner", "right", S(b), S(kb), condition=cond).collect(stream)
        assert sorted(j.column("row").to_pylist()) == rows
        j = BroadcastHashJoinExec(["k"], ["row"], "inner", "right", S(kb), FilterExec(cond, S(b))).collect(stream)
        assert sorted(j.column("row").to_pylist()) == rows
        e = ExpandExec([[Length(col("s"))], [OctetLength(col("s"))]], ["l"], S(b)).collect(stream)
        assert e.column("l").to_pylist()[0::2] == lens
        # Length over a binary column counts bytes, as Spark's Length over BinaryType does
        bv = [None, b"", "é日".encode(), b"\xff\xfe\x80"]
        bb = _scan(pa.table({"s": pa.array(bv, pa.binary())}), stream)
        try:
            assert ProjectExec([("l", Length(col("s")))], S(bb)).collect(stream).column("l").to_pylist() == [None, 0, 5, 3]
        finally:
            bb.close()
    finally:
        b.close()
        kb.close()


def test_project_filter_and_keys(gpu, stream):
    from spark_b200.execution import (BroadcastHashJoinExec, FilterExec, HashAggregateExec, LocalTableScanExec, ProjectExec, SortExec)
    from spark_b200.expressions import Concat, Count, In, Length, Literal, SortOrder, StartsWith, StringTrim, Substring, Sum, col
    S = LocalTableScanExec
    n = 30_007
    vals = random_strings(n, 21, ill=False)
    x = np.random.default_rng(3).integers(-50, 50, n).astype(np.int64)
    t = pa.table({"s": _binary_string(vals), "x": x})
    b = _scan(t, stream)
    try:
        ex = [("a", col("x") * Literal(2)), ("p", Substring(col("s"), 1, 2)), ("s", col("s")), ("l", Length(Substring(col("s"), 2, 3))),
              ("c", Concat(col("s"), "#"))]
        conds = [In(Substring(col("s"), 1, 1), ["a", "é", "😀"]), Concat(col("s"), "x").eq("ax"), StartsWith(StringTrim(col("s")), "Z") & (col("x") > Literal(0))]
        rows_of = [lambda r: vals[r] is not None and O.substring_sql(vals[r], 1, 1) in (b"a", "é".encode(), "😀".encode()),
                   lambda r: vals[r] == b"a",
                   lambda r: vals[r] is not None and O.trim(vals[r]).startswith(b"Z") and x[r] > 0]
        for cond, keep in zip(conds, rows_of):
            rows = [r for r in range(n) if keep(r)]
            for plan in (ProjectExec(ex, FilterExec(cond, S(b))), ProjectExec(ex, ProjectExec(["s", "x"], FilterExec(cond, S(b))))):
                got = plan.collect(stream)
                assert got.column_names == ["a", "p", "s", "l", "c"]
                assert got.column("a").to_pylist() == [int(x[r]) * 2 for r in rows]
                assert_column(got.column("p"), [O.substring_sql(vals[r], 1, 2) for r in rows])
                assert_column(got.column("s"), [vals[r] for r in rows])
                assert got.column("l").to_pylist() == [O.length(O.substring_sql(vals[r], 2, 3)) for r in rows]
                assert_column(got.column("c"), [O.concat(vals[r], b"#") for r in rows])
            f = FilterExec(cond, S(b)).collect(stream)
            assert f.column_names == ["s", "x"] and f.column("x").to_pylist() == [int(x[r]) for r in rows]
        # a string-function result as GROUP BY, join and ORDER BY key through a ProjectExec below
        keyed = ProjectExec([("k", Substring(col("s"), 1, 1)), ("x", col("x"))], S(b))
        agg = HashAggregateExec(["k"], [(Count(), "n"), (Sum(col("x")), "sx")], keyed).collect(stream)
        want = {}
        for r in range(n):
            k = O.substring_sql(vals[r], 1, 1)
            c, sx = want.get(k, (0, 0))
            want[k] = (c + 1, sx + int(x[r]))
        ks = agg.column("k").cast(pa.binary()).to_pylist()
        assert dict(zip(ks, zip(agg.column("n").to_pylist(), agg.column("sx").to_pylist()))) == want
        srt = SortExec([SortOrder("k"), SortOrder("x")], keyed).collect(stream)
        pairs = sorted(((O.substring_sql(vals[r], 1, 1), int(x[r])) for r in range(n)), key=lambda p: (p[0] is not None, p[0] or b"", p[1]))
        assert list(zip(srt.column("k").cast(pa.binary()).to_pylist(), srt.column("x").to_pylist())) == pairs
        dim = pa.table({"code": _binary_string([c.encode() for c in ("a", "é", "日", "😀")]), "w": np.arange(4, dtype=np.int64)})
        db = _scan(dim, stream)
        try:
            j = BroadcastHashJoinExec(["k"], ["code"], "inner", "right", keyed, S(db)).collect(stream)
            codes = {c.encode(): i for i, c in enumerate(("a", "é", "日", "😀"))}
            want = sorted((int(x[r]), codes[O.substring_sql(vals[r], 1, 1)]) for r in range(n) if O.substring_sql(vals[r], 1, 1) in codes)
            assert sorted(zip(j.column("x").to_pylist(), j.column("w").to_pylist())) == want
        finally:
            db.close()
    finally:
        b.close()


def test_tpch_q22_shape(gpu, stream):
    """Q22: customers whose phone country code is in a list, with a balance above the average positive balance of those codes and
    no orders, grouped and ordered by the code."""
    from spark_b200.execution import (BroadcastHashJoinExec, FilterExec, HashAggregateExec, LocalTableScanExec, ProjectExec, SortExec)
    from spark_b200.expressions import Average, Count, In, Literal, SortOrder, Substring, Sum, col
    S = LocalTableScanExec
    rng = np.random.default_rng(22)
    nc, no = 150_000, 600_000
    nation = rng.integers(0, 25, nc)
    phones = ["%02d-%03d-%03d-%04d" % (k + 10, a, b_, c) for k, a, b_, c in
              zip(nation, rng.integers(100, 1000, nc), rng.integers(100, 1000, nc), rng.integers(1000, 10000, nc))]
    bal = np.round(rng.uniform(-999.99, 9999.99, nc), 2)
    custkey = np.arange(1, nc + 1, dtype=np.int64)
    o_cust = rng.choice(custkey[custkey % 3 != 0], no)
    cust = pa.table({"c_custkey": custkey, "c_phone": pa.array(phones, pa.string()), "c_acctbal": bal})
    orders = pa.table({"o_custkey": o_cust})
    codes = ["13", "31", "23", "29", "30", "18", "17"]
    cb, ob = _scan(cust, stream), _scan(orders, stream)
    try:
        incodes = In(Substring(col("c_phone"), 1, 2), codes)
        avg = HashAggregateExec([], [(Average(col("c_acctbal")), "avg")], FilterExec(incodes & (col("c_acctbal") > Literal(0.0)), S(cb))).collect(stream)
        avg_bal = avg.column("avg").to_pylist()[0]
        sel = ProjectExec([("cntrycode", Substring(col("c_phone"), 1, 2)), ("c_acctbal", col("c_acctbal")), ("c_custkey", col("c_custkey"))],
                          FilterExec(incodes & (col("c_acctbal") > Literal(float(avg_bal))), S(cb)))
        anti = BroadcastHashJoinExec(["c_custkey"], ["o_custkey"], "left_anti", "right", sel, S(ob))
        agg = HashAggregateExec(["cntrycode"], [(Count(), "numcust"), (Sum(col("c_acctbal")), "totacctbal")], anti)
        got = SortExec([SortOrder("cntrycode")], agg).collect(stream)
        # numpy / pyarrow answer
        cc = np.array([p[:2] for p in phones])
        inm = np.isin(cc, codes)
        want_avg = bal[inm & (bal > 0)].mean()
        assert abs(avg_bal - want_avg) <= 1e-9 * abs(want_avg)
        has_order = np.zeros(nc + 1, bool)
        has_order[o_cust] = True
        keep = inm & (bal > avg_bal) & ~has_order[custkey]
        want_codes = sorted(set(cc[keep]))
        assert got.column("cntrycode").to_pylist() == want_codes
        assert got.column("numcust").to_pylist() == [int(np.sum(keep & (cc == c))) for c in want_codes]
        for g, c in zip(got.column("totacctbal").to_pylist(), want_codes):
            assert abs(g - bal[keep & (cc == c)].sum()) <= 1e-6
    finally:
        cb.close()
        ob.close()
