"""A plain reference for aggregate functions over every value type, and the data sets that exercise them (helper module, not
a test file).

`expected()` computes COUNT / COUNT(*) / MIN / MAX / SUM / AVG group by group from the raw storage values, without the C oracle:

- COUNT is exact.  Integer SUM adds in uint64, which is the Python integer sum reduced by `wrap64` (Spark's non-ANSI long SUM).
- A floating SUM or AVG (and an integer AVG, whose terms Spark widens to double) is bit-exact when every term is a finite
  quarter-integer and the group's sum of |x| stays below 2^50: every partial sum is then exact in any order, so the sum is the
  exact sum and AVG is one correctly rounded division of it, as in Spark and `__ddiv_rn`.  A group of two or more copies of one
  value whose double overflows (float64 MAX) sums to that infinity in any order.  Every other group is checked with
  `float_sums.check_sum` / `check_avg` against its terms.
- Decimal SUM / AVG: Python integers, NULL past the result precision, HALF_UP (restating `oracle.decimal_aggregate`).
- MIN / MAX order values like SQLOrderingUtil (NaN largest and equal to every NaN, -0.0 == 0.0, false < true, decimals by unscaled
  value).  Spark keeps the first extreme it meets (`reassignIfSmaller` keeps the incumbent on ties); the engine returns the
  extreme's own bits with two documented exceptions, which `engine=True` applies and records in `Expected.deviations`:
    1. ZERO_SIGNS: the extreme is a zero and both signs occur among the group's zeros: MIN is -0.0, MAX is +0.0;
    2. CANONICAL_NAN: the extreme is NaN: the canonical NaN (0x7FF8000000000000 / 0x7FC00000).
"""
import math

import numpy as np
import pyarrow as pa

from float_sums import _special, check_avg, check_sum
from test_gpu_key_types import TYPES, make_array, raw_bits, specials

INTEGRAL = ("int8", "int16", "int32", "int64")
FLOATS = ("float32", "float64")
DECIMALS = ("dec7_2", "dec18_0")
ZERO_SIGNS, CANONICAL_NAN = 1, 2
CANON = {"float32": 0x7FC00000, "float64": 0x7FF8000000000000}
SIGN = {"float32": 0x80000000, "float64": 0x8000000000000000}
_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def functions(tname):
    """The aggregate functions Spark's analyser accepts over a column of this type."""
    f = ["count", "count_star", "min", "max"]
    if tname in INTEGRAL + FLOATS + DECIMALS:
        f += ["sum", "avg"]
    return f


def _dec(p, s):
    return pa.decimal128(min(p, 38), s)


def result_type(func, tname):
    t = TYPES[tname]
    if func in ("count", "count_star"):
        return pa.int64()
    if func in ("min", "max"):
        return t
    if tname in DECIMALS:
        return _dec(t.precision + 10, t.scale) if func == "sum" else _dec(t.precision + 4, t.scale + 4)
    return pa.int64() if func == "sum" and tname in INTEGRAL else pa.float64()


def buffer_types(func, tname):
    """[(suffix, type)] of a Partial aggregate's buffer columns (Sum.scala, Average.scala, Count.scala, Min / Max.scala)."""
    t = TYPES[tname]
    if func in ("count", "count_star"):
        return [("#count", pa.int64())]
    if func in ("min", "max"):
        return [("#val", t)]
    if tname in DECIMALS:
        second = ("#isEmpty", pa.bool_()) if func == "sum" else ("#count", pa.int64())
        return [("#sum", _dec(t.precision + 10, t.scale)), second]
    if func == "sum":
        return [("#sum", result_type("sum", tname))]
    return [("#sum", pa.float64()), ("#count", pa.int64())]


def storage(arr, tname):
    """(values, valid) of an Arrow column: the storage values (unscaled longs for decimals, days / microseconds for dates and
    timestamps, 0 / 1 for bool), taken from the raw bits so that NaN payloads survive."""
    valid, words = raw_bits(arr)
    dt = specials(tname).dtype
    return words[0].astype(_UNSIGNED[dt.itemsize]).view(dt), valid


def storage_bits(values):
    return np.ascontiguousarray(values).view(_UNSIGNED[values.dtype.itemsize]).astype(np.uint64)


# ------------------------------------------------------------------------------------------------ grouping
def group_ids(table, key_cols):
    """(gid per row, number of groups, first row of each group): groups numbered in order of first occurrence.  Keys are
    compared by validity and raw bits (integer and date keys; float keys would need NormalizeFloatingNumbers first)."""
    n = table.num_rows
    if not key_cols:
        return np.zeros(n, np.int64), 1, np.zeros(1, np.int64)
    parts = []
    for k in key_cols:
        assert not pa.types.is_floating(table.schema.field(k).type), "float grouping keys are not handled by this reference"
        valid, words = raw_bits(table.column(k))
        parts.append(valid.astype(np.uint64))
        parts.extend(words)
    if n == 0:
        return np.zeros(0, np.int64), 0, np.zeros(0, np.int64)
    mat = np.stack(parts, axis=1)
    _, first, inv = np.unique(mat, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    remap = np.empty(len(order), np.int64)
    remap[order] = np.arange(len(order))
    return remap[inv.reshape(-1)], len(order), first[order]


# ------------------------------------------------------------------------------------------------ the reference
class Expected:
    """The expected output table (keys ++ aggregate columns, groups in order of first occurrence) plus:
    approx[col] = {row: (check, terms, label)}: cells checked with float_sums.check_sum / check_avg against their terms (the
    table holds the correctly rounded answer there);
    deviations[col] = int array per row: ZERO_SIGNS / CANONICAL_NAN where exception 1 / 2 decided the MIN / MAX bits;
    first_seen[col] = Spark's first-seen MIN / MAX bits (uint64) per row, for comparison with the oracle."""

    def __init__(self):
        self.names, self.arrays = [], []
        self.approx, self.deviations, self.first_seen = {}, {}, {}

    def add(self, name, arr):
        self.names.append(name)
        self.arrays.append(arr)

    @property
    def table(self):
        return pa.table(dict(zip(self.names, self.arrays)))


def _dec_array(t, ints, valid):
    """decimal128 array from Python integers of any size (two's complement, 16 bytes each)."""
    n = len(ints)
    raw = b"".join(int(v if ok else 0).to_bytes(16, "little", signed=True) for v, ok in zip(ints, valid))
    vb = None if all(valid) else pa.py_buffer(np.packbits(np.asarray(valid, bool), bitorder="little").tobytes())
    return pa.Array.from_buffers(t, n, [vb, pa.py_buffer(raw)])


def _int_array(t, vals, valid):
    return pa.Array.from_buffers(t, len(vals), [None if valid.all() else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()),
                                                pa.py_buffer(np.ascontiguousarray(vals).tobytes())])


def _counts(gid, valid, ng):
    return np.bincount(gid[valid], minlength=ng).astype(np.int64)


def _group_sums_exact(gid, x, ng):
    """Exact per-group sums of int64 storage values as Python integers (each value split into 32-bit halves so that the
    per-half sums fit int64 for any group below 2^31 rows)."""
    lo = (x & 0xFFFFFFFF).astype(np.int64)
    hi = x >> 32
    slo, shi = np.zeros(ng, np.int64), np.zeros(ng, np.int64)
    np.add.at(slo, gid, lo)
    np.add.at(shi, gid, hi)
    return [int(h) * (1 << 32) + int(l) for h, l in zip(shi.tolist(), slo.tolist())]


def _float_sums(gid, xs, ng, cnt, avg, what):
    """(values float64, approx {row: (check, terms, label)}) of SUM / AVG over double terms xs (NULLs removed), see the module
    doc."""
    fin = np.isfinite(xs)
    q = np.zeros(len(xs), np.float64)
    q[fin] = xs[fin] * 4
    quarter = fin & (q == np.floor(q)) & (np.abs(xs) <= 2.0 ** 40)
    bad = np.bincount(gid[~quarter], minlength=ng)
    mag = np.zeros(ng)
    np.add.at(mag, gid[quarter], np.abs(xs[quarter]))
    exact = (bad == 0) & (mag <= 2.0 ** 50)
    s4 = np.zeros(ng, np.int64)
    np.add.at(s4, gid[quarter], q[quarter].astype(np.int64))
    with np.errstate(invalid="ignore", divide="ignore"):
        sums = s4.astype(np.float64) / 4          # exact: |s4| < 2^53
        out = sums / np.maximum(cnt, 1) if avg else sums
    approx = {}
    rows = np.nonzero(~exact & (cnt > 0))[0]
    if len(rows):
        order = np.argsort(gid, kind="stable")
        sg = gid[order]
        starts = np.searchsorted(sg, rows)
        ends = np.searchsorted(sg, rows, side="right")
        for g, a, b in zip(rows.tolist(), starts.tolist(), ends.tolist()):
            terms = xs[order[a:b]]
            if len(terms) > 1 and np.all(terms == terms[0]) and np.isfinite(terms[0]) and np.isinf(terms[0] + terms[0]):
                out[g] = terms[0] + terms[0]                # v + v overflows: every order reaches that infinity
                continue
            approx[g] = (check_avg if avg else check_sum, terms.tolist(), "%s group %d" % (what, g))
            sp = _special(terms.tolist())                   # the table holds the correctly rounded answer there
            out[g] = sp if sp is not None else math.fsum(terms.tolist()) / (len(terms) if avg else 1)
    return out, approx


def _order_ranks(vals, tname):
    """int64 rank per value in SQLOrderingUtil's order: NaN largest and equal to every NaN, -0.0 == 0.0."""
    if tname in FLOATS:
        x = vals.astype(np.float64)
        x = np.where(x == 0, 0.0, x)                    # -0.0 == 0.0
        uniq = np.unique(x)                             # sorted, NaN last, all NaNs one entry
        return np.searchsorted(uniq, x).astype(np.int64)
    return vals.astype(np.int64)


def _minmax(gid, vals, valid, ng, tname, is_max, engine):
    """(bits uint64 per group, seen bool, deviation kind per group, Spark's first-seen bits per group)."""
    vg, xv = gid[valid], vals[valid]
    rank = _order_ranks(xv, tname)
    best = np.full(ng, np.iinfo(np.int64).min if is_max else np.iinfo(np.int64).max, np.int64)
    (np.maximum if is_max else np.minimum).at(best, vg, rank)
    seen = np.bincount(vg, minlength=ng) > 0
    hit = rank == best[vg]
    hit_g = vg[hit]
    bits = storage_bits(xv)[hit]
    ug, first = np.unique(hit_g, return_index=True)       # rows are in table order: the first extreme of each group
    first_seen = np.zeros(ng, np.uint64)
    first_seen[ug] = bits[first]
    out, dev = first_seen.copy(), np.zeros(ng, np.int64)
    if tname in FLOATS:
        xh = xv[hit].astype(np.float64)
        nan_g = np.unique(hit_g[np.isnan(xh)])
        zero = xh == 0
        neg = np.zeros(ng, bool)
        pos = np.zeros(ng, bool)
        neg[hit_g[zero & (bits == SIGN[tname])]] = True
        pos[hit_g[zero & (bits == 0)]] = True
        both = np.nonzero(neg & pos)[0]
        dev[both] = ZERO_SIGNS
        dev[nan_g] = CANONICAL_NAN
        if engine:
            out[both] = 0 if is_max else SIGN[tname]
            out[nan_g] = CANON[tname]
    return out, seen, dev, first_seen


def _bits_array(t, tname, bits, valid):
    dt = specials(tname).dtype
    vals = bits.astype(_UNSIGNED[dt.itemsize]).view(dt)
    return make_array(t, vals, valid)


def expected(table, key_cols, aggs, mode="complete", engine=True):
    """Expected output of HashAggregateExec(key_cols, aggs) over `table` in `mode` ('complete' or 'partial': keys ++
    buffers).  aggs = [(func, column, out_name)]; the value columns' types are named by TYPE_NAMES (see `type_name`)."""
    with np.errstate(invalid="ignore", over="ignore"):
        return _expected(table, key_cols, aggs, mode, engine)


def _expected(table, key_cols, aggs, mode, engine):
    gid, ng, first = group_ids(table, key_cols)
    e = Expected()
    for k in key_cols:
        e.add(k, table.column(k).combine_chunks().take(pa.array(first)))
    for func, cname, name in aggs:
        if func == "count_star":
            cnt = np.bincount(gid, minlength=ng).astype(np.int64)
            e.add(name + "#count" if mode == "partial" else name, pa.array(cnt, pa.int64()))
            continue
        tname = type_name(table.schema.field(cname).type)
        vals, valid = storage(table.column(cname), tname)
        cnt = _counts(gid, valid, ng)
        seen = cnt > 0
        if func == "count":
            e.add(name + "#count" if mode == "partial" else name, pa.array(cnt, pa.int64()))
            continue
        if func in ("min", "max"):
            bits, seen_, dev, fs = _minmax(gid, vals, valid, ng, tname, func == "max", engine)
            col = name + "#val" if mode == "partial" else name
            e.add(col, _bits_array(TYPES[tname], tname, bits, seen_))
            e.deviations[col], e.first_seen[col] = dev, fs
            continue
        gv, xv = gid[valid], vals[valid]
        if tname in DECIMALS:
            t = TYPES[tname]
            sums = _group_sums_exact(gv, xv.astype(np.int64), ng)
            sum_t = result_type("sum", tname)
            if mode == "partial":
                e.add(name + "#sum", _dec_array(sum_t, [s if c else 0 for s, c in zip(sums, cnt.tolist())], [True] * ng))
                if func == "sum":
                    e.add(name + "#isEmpty", pa.array(~seen, pa.bool_()))
                else:
                    e.add(name + "#count", pa.array(cnt, pa.int64()))
                continue
            if func == "sum":
                ok = [c > 0 and abs(s) < 10 ** sum_t.precision for s, c in zip(sums, cnt.tolist())]
                e.add(name, _dec_array(sum_t, sums, ok))
            else:
                avg_t = result_type("avg", tname)
                res, ok = [], []
                for s, c in zip(sums, cnt.tolist()):
                    if c == 0:
                        res.append(0)
                        ok.append(False)
                        continue
                    q, r = divmod(abs(s) * 10 ** 4, c)
                    q += 2 * r >= c                       # HALF_UP
                    q = -q if s < 0 else q
                    res.append(q)
                    ok.append(abs(q) < 10 ** avg_t.precision)
                e.add(name, _dec_array(avg_t, res, ok))
            continue
        if func == "sum" and tname in INTEGRAL:
            acc = np.zeros(ng, np.uint64)
            np.add.at(acc, gv, xv.astype(np.int64).view(np.uint64))   # mod 2^64: wrap64 of the exact sum
            e.add(name + "#sum" if mode == "partial" else name, _int_array(pa.int64(), acc.view(np.int64), seen))
            continue
        xs = xv.astype(np.float64)                        # float32 and integer terms widened to double per term
        if func == "sum":
            s, approx = _float_sums(gv, xs, ng, cnt, False, "sum(%s)" % cname)
            col = name + "#sum" if mode == "partial" else name
            e.add(col, _int_array(pa.float64(), s, seen))
            e.approx[col] = approx
            continue
        if mode == "partial":                             # Average's buffers: sum (0.0 when empty, never NULL), count
            s, approx = _float_sums(gv, xs, ng, cnt, False, "avg(%s)#sum" % cname)
            e.add(name + "#sum", _int_array(pa.float64(), s, np.ones(ng, bool)))
            e.add(name + "#count", pa.array(cnt, pa.int64()))
            e.approx[name + "#sum"] = approx
            continue
        a, approx = _float_sums(gv, xs, ng, cnt, True, "avg(%s)" % cname)
        e.add(name, _int_array(pa.float64(), a, seen))
        e.approx[name] = approx
    return e


def type_name(t):
    for k, v in TYPES.items():
        if v == t:
            return k
    raise KeyError(t)


# ------------------------------------------------------------------------------------------------ comparison
def _key_order(table, nkeys):
    keys = []
    for i in range(nkeys):
        valid, words = raw_bits(table.column(i))
        keys.append(valid)
        keys.extend(words)
    return np.lexsort(keys[::-1]) if keys else np.arange(table.num_rows)


def assert_expected(got, exp, nkeys):
    """`got` equals `exp` bit for bit: column names, types, row count, keys, validity and raw bits; cells in exp.approx are
    checked with float_sums against their terms instead of bit for bit."""
    want = exp.table
    assert got.column_names == want.column_names, (got.column_names, want.column_names)
    for i in range(want.num_columns):
        assert got.schema.field(i).type == want.schema.field(i).type, \
            "column %s: type %s != %s" % (want.column_names[i], got.schema.field(i).type, want.schema.field(i).type)
    assert got.num_rows == want.num_rows, "row count %d != %d" % (got.num_rows, want.num_rows)
    gp, wp = _key_order(got, nkeys), _key_order(want, nkeys)
    for i, name in enumerate(want.column_names):
        gv, gw = raw_bits(got.column(i))
        wv, ww = raw_bits(want.column(i))
        gv, wv = gv[gp], wv[wp]
        bad = np.nonzero(gv != wv)[0]
        assert len(bad) == 0, "column %s row %d: valid %s vs %s" % (name, wp[bad[0]], gv[bad[0]], wv[bad[0]])
        skip = np.zeros(want.num_rows, bool)
        approx = exp.approx.get(name, {})
        if approx:
            at = np.empty(want.num_rows, np.int64)
            at[wp] = np.arange(want.num_rows)             # expected row -> position in the aligned order
            gvals = got.column(i).combine_chunks().to_numpy(zero_copy_only=False)[gp]
            for row, (check, terms, what) in approx.items():
                check(float(gvals[at[row]]), terms, what)
                skip[at[row]] = True
        for a, b in zip(gw, ww):
            a, b = a[gp], b[wp]
            bad = np.nonzero((a != b) & ~skip)[0]
            assert len(bad) == 0, "column %s row %d: bits %#x vs %#x (%d rows differ)" % (
                name, wp[bad[0]], int(a[bad[0]]), int(b[bad[0]]), len(bad))


# ------------------------------------------------------------------------------------------------ data
def type_extremes(tname):
    """(MIN, MAX) storage values of a type: integer limits, decimal +-(10^p - 1), false / true, float -MAX / MAX."""
    if tname == "bool":
        return 0, 1
    if tname in DECIMALS:
        top = 10 ** TYPES[tname].precision - 1
        return -top, top
    if tname in FLOATS:
        m = np.finfo(np.float32 if tname == "float32" else np.float64).max
        return -m, m
    info = np.iinfo(specials(tname).dtype)
    return int(info.min), int(info.max)


def _floats(tname, bits):
    dt = np.float32 if tname == "float32" else np.float64
    return np.array(bits, dtype=_UNSIGNED[np.dtype(dt).itemsize]).view(dt)


def special_groups(tname):
    """[(label, storage values, valid)]: the designated groups every keyed data set starts with."""
    dt = specials(tname).dtype
    lo, hi = type_extremes(tname)
    minus_one = 1 if tname == "bool" else -1
    g = [("all_null", np.zeros(3, dt), np.zeros(3, bool)),
         ("single", np.array([1], dt), np.ones(1, bool)),
         ("only_min", np.array([lo] * 3, dt), np.ones(3, bool)),
         ("only_max", np.array([hi] * 3, dt), np.ones(3, bool)),
         ("only_minus_one", np.array([minus_one] * 3, dt), np.ones(3, bool)),
         ("extremes", np.array([lo, 0, minus_one, hi] if tname not in FLOATS else [lo, 0, -1, 1], dt), np.ones(4, bool)),
         ("with_nulls", np.array([minus_one, 0, 1, 0], dt), np.array([True, False, True, False]))]
    if tname in FLOATS:
        if tname == "float64":
            nan_only, nan_inf = [0xFFF8000000000000, 0x7FF4000000000000, 0x7FF0000000000001], [0xFFF8000000000001]
            tiny = [0x1]
        else:
            nan_only, nan_inf = [0xFFC00000, 0x7FC00001, 0x7F800001], [0xFFC00001]
            tiny = [0x1]
        g += [("zeros_pos_first", np.array([0.0, -0.0, -0.0, 0.0], dt), np.ones(4, bool)),
              ("zeros_neg_first", np.array([-0.0, 0.0, -2.5], dt), np.ones(3, bool)),
              ("only_neg_zero", np.array([-0.0, -0.0], dt), np.ones(2, bool)),
              ("only_nan", _floats(tname, nan_only), np.ones(3, bool)),
              ("nan_inf", np.concatenate([_floats(tname, nan_inf), np.array([np.inf, -np.inf, 1.5], dt)]), np.ones(4, bool)),
              ("subnormal", _floats(tname, tiny), np.ones(1, bool))]
    return g


def ordinary_values(tname, k, rng):
    """Random values of a type: full range for narrow integers and dates, |x| < 2^31 for int64 (AVG stays exact),
    full range for timestamps and decimals, quarter-integers for floats."""
    dt = specials(tname).dtype
    if tname == "bool":
        return rng.integers(0, 2, k).astype(dt)
    if tname in FLOATS:
        return (rng.integers(-4000, 4000, k) / 4.0).astype(dt)
    if tname == "int64":
        return rng.integers(-(1 << 31), 1 << 31, k).astype(dt)
    lo, hi = type_extremes(tname)
    return rng.integers(lo, hi, k, dtype=np.int64, endpoint=True).astype(dt)


LAYOUTS = ("none", "dict7", "g31", "g32", "g33", "smem60k", "wide")


def value_table(tname, n, layout, validity, seed):
    """n rows of keys ++ a value column "v" of type tname.

    layout: none (no keys), dict7 (int32 key, 7 groups), g31 / g32 / g33 (int32 key, exactly that many groups when n is large
    enough), smem60k (int32 key, ~60 000 groups), wide (nullable int64 + int32 key).  Keyed layouts but dict7 start with the
    special_groups() of the type, each under its own key.  validity: none (no validity buffer), nulls (10 % NULL, plus the
    all-NULL group), allnull.  Rows are shuffled."""
    rng = np.random.default_rng(seed)
    dt = specials(tname).dtype
    vals, valid, grp = [], [], []
    nspecial = 0
    if layout not in ("none", "dict7"):
        for i, (label, v, ok) in enumerate(special_groups(tname)):
            if validity == "none" and label == "all_null":
                continue
            vals.append(v)
            valid.append(ok)
            grp.append(np.full(len(v), -1 - i, np.int64))
            nspecial += 1
    vals = np.concatenate(vals)[:n] if vals else np.zeros(0, dt)
    valid = np.concatenate(valid)[:n] if valid else np.zeros(0, bool)
    grp = np.concatenate(grp)[:n] if grp else np.zeros(0, np.int64)
    k = n - len(vals)
    ng = {"none": 1, "dict7": 7, "g31": 31 - nspecial, "g32": 32 - nspecial, "g33": 33 - nspecial, "smem60k": 60_000, "wide": 3000}[layout]
    og = rng.integers(0, ng, k)
    og[:min(k, ng)] = np.arange(min(k, ng))              # every ordinary group present when there are rows enough
    vals = np.concatenate([vals, ordinary_values(tname, k, rng)])
    valid = np.concatenate([valid, rng.random(k) >= 0.1])
    grp = np.concatenate([grp, og])
    perm = rng.permutation(n)
    vals, valid, grp = vals[perm], valid[perm], grp[perm]
    if validity == "none":
        valid = None
    elif validity == "allnull":
        valid = np.zeros(n, bool)
    cols = {}
    if layout == "wide":
        pool = np.array([np.iinfo(np.int64).min, -1, np.iinfo(np.int64).max, 0, 1, 1 << 40], np.int64)
        k0 = np.where(grp < 0, grp * 7919, pool[np.abs(grp) % len(pool)])
        k0_valid = (grp < 0) | (rng.random(n) >= 0.05)
        cols["k0"] = make_array("int64", k0, k0_valid)
        cols["k1"] = make_array("int32", (grp // len(pool)).astype(np.int32))
    elif layout != "none":
        cols["k"] = make_array("int32", grp.astype(np.int32))
    cols["v"] = make_array(tname, vals, valid)
    return pa.table(cols)


def key_names(layout):
    return [] if layout == "none" else (["k0", "k1"] if layout == "wide" else ["k"])


def all_aggs(tname, col="v", prefix=""):
    return [(f, col, prefix + f) for f in functions(tname)]
