"""Host-only checks of the aggregate value reference (tests/aggregate_values.py): it agrees with the C oracle wherever Spark's
answer is deterministic, its data sets hold what they claim, and its comparison catches a single flipped bit."""
import numpy as np
import pyarrow as pa
import pytest

import aggregate_values as A
from oracle import oracle as O
from test_gpu_key_types import TYPE_NAMES, TYPES, make_array, raw_bits

F32_QUIET = 0x00400000


def _oracle(t, keys, tname):
    """The C oracle's answer for every function of the type, columns named like A.all_aggs."""
    aggs = A.all_aggs(tname)
    if tname in A.DECIMALS:
        dec = O.decimal_aggregate(t, keys, [a for a in aggs if a[0] != "count_star"])
        star = O.hash_aggregate(t, keys, [a for a in aggs if a[0] == "count_star"])
        return O.take_table(star, np.arange(star.num_rows)), dec
    return O.hash_aggregate(t, keys, aggs), None


def _aligned(table, keys):
    return A._key_order(table.select(keys), len(keys)) if keys else np.arange(table.num_rows)


def _compare_with_oracle(t, keys, tname):
    """Bit-exact agreement of the engine reference with the oracle outside exception cells; returns, per exception kind, how
    many cells it decided and in how many of them the bits differ from Spark's first-seen answer."""
    e = A.expected(t, keys, A.all_aggs(tname))
    want = e.table
    main, dec = _oracle(t, keys, tname)
    wp = _aligned(want, keys)
    found = {A.ZERO_SIGNS: [0, 0], A.CANONICAL_NAN: [0, 0]}
    for func, _, name in A.all_aggs(tname):
        src = dec if dec is not None and name in dec.column_names else main
        op = _aligned(src, keys)
        assert src.num_rows == want.num_rows
        oc, wc = src.column(name).combine_chunks(), want.column(name).combine_chunks()
        if oc.type != wc.type:            # the oracle returns MIN / MAX of timestamps as plain longs
            assert func in ("min", "max") and oc.type == pa.int64(), (name, oc.type, wc.type)
            ov, _ = A.storage(oc, "int64")
            oc = make_array(wc.type, ov, np.asarray(oc.is_valid()))
        ovalid, ow = raw_bits(oc)
        wvalid, ww = raw_bits(wc)
        assert np.array_equal(ovalid[op], wvalid[wp]), name
        skip = np.zeros(want.num_rows, bool)
        for row, (check, terms, what) in e.approx.get(name, {}).items():
            pos = int(np.nonzero(wp == row)[0][0])
            check(float(oc[int(op[pos])].as_py()), terms, what)        # the oracle's sequential sum meets the same bound
            skip[pos] = True
        dev = e.deviations.get(name)
        if dev is not None:
            for pos in np.nonzero(dev[wp] > 0)[0]:
                kind = int(dev[wp][pos])
                fs = int(e.first_seen[name][wp][pos])
                got = int(ow[0][op][pos])
                if tname == "float32" and kind == A.CANONICAL_NAN:
                    fs |= F32_QUIET                     # the oracle widens float32 to double, which quiets a signalling NaN
                assert got == fs, "%s: oracle %#x, first seen %#x" % (name, got, fs)
                found[kind][0] += 1
                found[kind][1] += int(ww[0][wp][pos]) != fs
                skip[pos] = True
        for a, b in zip(ow, ww):
            bad = np.nonzero((a[op] != b[wp]) & ~skip)[0]
            assert len(bad) == 0, "%s: oracle %#x, reference %#x" % (name, int(a[op][bad[0]]), int(b[wp][bad[0]]))
    return found


@pytest.mark.parametrize("layout", ["none", "dict7", "g33", "wide"])
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_reference_agrees_with_the_oracle(tname, layout):
    total = {A.ZERO_SIGNS: [0, 0], A.CANONICAL_NAN: [0, 0]}
    for i, validity in enumerate(("none", "nulls", "allnull")):
        t = A.value_table(tname, 4097, layout, validity, seed=i)
        for kind, (n, diff) in _compare_with_oracle(t, A.key_names(layout), tname).items():
            total[kind][0] += n
            total[kind][1] += diff
    if tname in A.FLOATS and layout in ("g33", "wide"):
        # per validity variant with values: MIN and MAX of zeros_pos_first and MAX of zeros_neg_first have zeros of both
        # signs (the shuffled row order decides which one Spark meets first), MIN and MAX of only_nan and MAX of nan_inf are
        # NaN, never the canonical one
        assert total[A.ZERO_SIGNS][0] == 6 and total[A.ZERO_SIGNS][1] > 0, total
        assert total[A.CANONICAL_NAN] == [6, 6], total
    else:
        assert total == {A.ZERO_SIGNS: [0, 0], A.CANONICAL_NAN: [0, 0]}, total


def test_reference_agrees_with_exact_integer_arithmetic():
    """Integer SUM is wrap64 of the Python sum; AVG of an exact group is float(Fraction(sum, count))."""
    from fractions import Fraction
    from float_sums import wrap64
    for tname in A.INTEGRAL:
        t = A.value_table(tname, 2000, "g33", "nulls", seed=5)
        e = A.expected(t, ["k"], [("sum", "v", "s"), ("avg", "v", "a")]).table
        vals, valid = A.storage(t.column("v"), tname)
        keys = t.column("k").to_numpy()
        for key, s, a in zip(e.column("k").to_pylist(), e.column("s").to_pylist(), e.column("a").to_pylist()):
            xs = [int(x) for x in vals[(keys == key) & valid]]
            assert s == (wrap64(sum(xs)) if xs else None)
            if xs and max(abs(x) for x in xs) < 2 ** 53:
                assert a == float(Fraction(sum(xs), len(xs)))


@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_data_sets_hold_what_they_claim(tname):
    lo, hi = A.type_extremes(tname)
    t = A.value_table(tname, 4097, "g33", "nulls", seed=1)
    keys = t.column("k").to_numpy()
    vals, valid = A.storage(t.column("v"), tname)
    groups = dict((label, i) for i, (label, _, _) in enumerate(A.special_groups(tname)))
    rows = {label: (vals[keys == -1 - i], valid[keys == -1 - i]) for label, i in groups.items()}
    assert len(np.unique(keys)) == 33
    v, ok = rows["all_null"]
    assert len(v) == 3 and not ok.any()
    assert len(rows["single"][0]) == 1 and rows["single"][1].all()
    for label, want in (("only_min", lo), ("only_max", hi)):
        v, ok = rows[label]
        assert len(v) == 3 and ok.all() and np.all(A.storage_bits(v) == A.storage_bits(np.array([want], v.dtype)))
    v, _ = rows["only_minus_one"]
    assert np.all(v == (1 if tname == "bool" else -1))
    if tname in ("int64", "timestamp"):          # the MAX / MIN accumulator identities after the X_SIGNED flip
        assert rows["only_min"][0][0] == np.iinfo(np.int64).min and rows["only_max"][0][0] == np.iinfo(np.int64).max
    if tname in A.FLOATS:
        bits = lambda label: A.storage_bits(rows[label][0])
        sign = A.SIGN[tname]
        assert set(bits("zeros_pos_first")) == {0, sign} and {0, sign} <= set(bits("zeros_neg_first"))
        assert set(bits("only_neg_zero")) == {sign}
        v = rows["only_nan"][0]
        assert np.isnan(v).all() and A.CANON[tname] not in set(bits("only_nan")) and len(set(bits("only_nan"))) == 3
        v = rows["nan_inf"][0]
        assert np.isnan(v).any() and np.isposinf(v).any() and np.isneginf(v).any()
        v = rows["subnormal"][0]
        assert 0 < abs(float(v[0])) < np.finfo(v.dtype).tiny
    # group counts and validity variants of every layout
    for layout, want in (("dict7", 7), ("g31", 31), ("g32", 32), ("g33", 33)):
        assert len(np.unique(A.value_table(tname, 4097, layout, "none", 0).column("k").to_numpy())) == want
    assert len(np.unique(A.value_table(tname, 100_003, "smem60k", "none", 0).column("k").to_numpy())) > 50_000
    assert A.value_table(tname, 4097, "wide", "nulls", 0).column("k0").null_count > 0
    assert A.value_table(tname, 4097, "g33", "none", 0).column("v").chunk(0).buffers()[0] is None
    assert A.value_table(tname, 4097, "g33", "allnull", 0).column("v").null_count == 4097


def _with_bits(table, name, row, flip=None, new_type=None):
    """A copy of `table` with the raw bits of one cell XOR-ed with `flip`, or column `name` relabelled as `new_type`."""
    cols = {}
    for n in table.column_names:
        arr = table.column(n).combine_chunks()
        if n == name:
            tname = A.type_name(arr.type)
            vals, valid = A.storage(arr, tname)
            vals = vals.copy()
            if flip is not None:
                b = A.storage_bits(vals)
                b[row] ^= flip
                vals = b.astype(A._UNSIGNED[vals.dtype.itemsize]).view(vals.dtype)
            arr = make_array(new_type or arr.type, vals, valid)
        cols[n] = arr
    return pa.table(cols)


def _row_of(exp, key):
    return int(np.nonzero(exp.table.column("k").to_numpy() == key)[0][0])


@pytest.mark.parametrize("case", ["zero_sign", "nan_payload", "int16_high_byte", "decimal_scale"])
def test_comparison_catches_one_flipped_bit(case):
    tname, col, label, flip, new_type = {
        "zero_sign": ("float64", "max", "zeros_neg_first", A.SIGN["float64"], None),
        "nan_payload": ("float32", "max", "only_nan", 1, None),
        "int16_high_byte": ("int16", "min", "only_max", 0x0100, None),
        "decimal_scale": ("dec7_2", "min", "extremes", None, pa.decimal128(7, 3)),
    }[case]
    t = A.value_table(tname, 500, "g33", "nulls", seed=2)
    exp = A.expected(t, ["k"], A.all_aggs(tname))
    A.assert_expected(exp.table, exp, 1)                 # the unmodified answer passes
    label_index = [lb for lb, _, _ in A.special_groups(tname)].index(label)
    bad = _with_bits(exp.table, col, _row_of(exp, -1 - label_index), flip, new_type)
    with pytest.raises(AssertionError):
        A.assert_expected(bad, exp, 1)


def test_result_and_buffer_types():
    assert A.result_type("sum", "int8") == pa.int64() and A.result_type("sum", "float32") == pa.float64()
    assert A.result_type("sum", "dec7_2") == pa.decimal128(17, 2) and A.result_type("avg", "dec18_0") == pa.decimal128(22, 4)
    assert A.result_type("min", "dec7_2") == pa.decimal128(7, 2) and A.result_type("max", "float32") == pa.float32()
    assert A.buffer_types("avg", "int16") == [("#sum", pa.float64()), ("#count", pa.int64())]
    assert A.buffer_types("sum", "dec18_0") == [("#sum", pa.decimal128(28, 0)), ("#isEmpty", pa.bool_())]
    assert A.functions("bool") == ["count", "count_star", "min", "max"] and "avg" in A.functions("dec7_2")
    assert all(A.type_name(TYPES[t]) == t for t in TYPE_NAMES)
