"""GPU parity for every aggregate function over every value type, BIT FOR BIT against the plain reference of
tests/aggregate_values.py: COUNT / COUNT(*) / MIN / MAX over bool, int8..int64, date32, timestamp, decimal(7, 2), decimal(18, 0),
float32 and float64, and SUM / AVG where Spark accepts them.

The value path is type-specific at every step (load_i64_batch widens each width, MIN / MAX map values to order-preserving words
and back, agg_emit_kernel narrows through store_typed, decimal results carry their precision and scale, decimal SUM / AVG go
through the limb rewrite of decimal.cu), so every type runs through every update kernel (dictionary tier, shared-memory tier,
generic, run-time specialised, automatic), every key layout, Partial / Final / PartialMerge and the batch-by-batch state.
"""
import functools

import numpy as np
import pyarrow as pa
import pytest

import aggregate_values as A
from test_gpu_key_types import AGG_ENV_IDS, AGG_ENVS, TYPE_NAMES, make_array, specials

pytestmark = pytest.mark.gpu

ENVS = AGG_ENVS + [{}]                  # ... and the automatic choice with default settings
ENV_IDS = AGG_ENV_IDS + ["auto"]


def _specs(aggs):
    from spark_b200.expressions import Average, Count, Max, Min, Sum, col
    fn = {"sum": Sum, "avg": Average, "count": Count, "min": Min, "max": Max}
    return [(Count() if f == "count_star" else fn[f](col(c)), name) for f, c, name in aggs]


def _batch(t, stream):
    from spark_b200.columnar import ColumnarBatch
    return ColumnarBatch.from_arrow(t, stream)


def _agg(t, keys, aggs, stream, mode="complete", cls=None):
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    cls = cls or HashAggregateExec
    return cls(keys, _specs(aggs), LocalTableScanExec(_batch(t, stream)), mode=mode).collect(stream)


def _env(sbconfig, env):
    for k, v in env.items():
        sbconfig(k, v)


def _check(t, keys, aggs, stream, mode="complete", want=None):
    got = _agg(t, keys, aggs, stream, mode)
    A.assert_expected(got, want or A.expected(t, keys, aggs, mode), len(keys))
    return got


@functools.lru_cache(maxsize=16)
def _case(tname, layout, n, validity, seed):
    """A data set and its expected Complete answer, shared by the update kernels that run it one after another."""
    t = A.value_table(tname, n, layout, validity, seed)
    return t, A.expected(t, A.key_names(layout), A.all_aggs(tname))


# ------------------------------------------------------------------------------------------------ 1. Complete, every kernel
# (n, validity): 4096 = 128 x 4 x 8 rows is the automatic "tiny" cut-over, 4097 the first row past it
RUNS = [(0, "nulls"), (1, "none"), (33, "allnull"), (4096, "nulls"), (4097, "none"), (100_003, "nulls"), (100_003, "allnull")]
# One-word layouts under every update kernel; the two-word layout runs the wide kernels whatever the tier or rtc setting.  The
# tier1 / tier2 / rtc settings compile kernels for each plan at run time, so they run the int32-key layouts (one plan, shared by
# dict7, g31_33 and smem60k) and rtc also the global one, NULL-free runs left out (test_default_settings_* compiles those).
LAYOUT_ENVS = ([(layout, env) for layout in ("dict7", "g31_33", "smem60k") for env in ENV_IDS] +
               [("none", "generic"), ("none", "rtc"), ("none", "auto"), ("wide", "auto")])


@pytest.mark.parametrize("layout,env", LAYOUT_ENVS)
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_complete_every_kernel(gpu, stream, sbconfig, tname, layout, env):
    """Every function of the type in one plan.  Key layouts: none (global), one int32 key with 7 groups (dictionary tier), 31 /
    32 / 33 groups (agg_emit_kernel's validity ballots over a partial last warp), ~60 000 groups (shared-memory table spilling
    to HBM, then the bypass), a nullable int64 + int32 key pair (two key words: the wide kernels).  Keyed layouts but dict7 hold
    the special groups (all-NULL, single row, only MIN / MAX / -1, both zero signs, non-canonical NaNs, NaN with +-inf)."""
    _env(sbconfig, ENVS[ENV_IDS.index(env)])
    for i, (n, validity) in enumerate(RUNS):
        if env in ("tier1", "tier2", "rtc") and validity == "none":
            continue
        lay = ("g31", "g32", "g33")[i % 3] if layout == "g31_33" else layout
        t, want = _case(tname, lay, n, validity, i)
        _check(t, A.key_names(lay), A.all_aggs(tname), stream, want=want)


@pytest.mark.parametrize("env", [ENVS[2], ENVS[4]], ids=["generic", "auto"])
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_global_aggregate_of_each_special_group(gpu, stream, sbconfig, tname, env):
    """Each special group alone as a global aggregate: one row, one to four values (the same groups meet every update kernel
    in test_complete_every_kernel's keyed layouts).  Pins the two documented MIN / MAX
    deviations: zeros of both signs give MIN -0.0 / MAX +0.0, a NaN extreme is the canonical NaN, and where one bit pattern
    reaches the extreme (only -0.0, a subnormal, one non-canonical NaN payload through MIN of NaNs) it comes back as it is."""
    _env(sbconfig, env)
    aggs = A.all_aggs(tname)
    for label, vals, valid in A.special_groups(tname):
        t = pa.table({"v": make_array(tname, vals, valid)})
        got = _check(t, [], aggs, stream)
        if label == "only_nan":
            assert A.storage_bits(A.storage(got.column("max"), tname)[0])[0] == A.CANON[tname]
        if label == "only_neg_zero":
            assert A.storage_bits(A.storage(got.column("max"), tname)[0])[0] == A.SIGN[tname]


@pytest.mark.parametrize("tname,validity", [("int8", "none"), ("int16", "nulls"), ("bool", "nulls"), ("float32", "none")])
def test_default_settings_specialise_narrow_values(gpu, stream, tname, validity):
    """Past agg_rtc_min_rows (2^20) the automatic mode runs kernels specialised for the plan: narrow value types must take
    them and answer bit for bit, with and without a validity buffer."""
    from spark_b200 import _capi as capi
    n = (1 << 20) + 7
    t = A.value_table(tname, n, "g33", validity, seed=11)
    _check(t, ["k"], A.all_aggs(tname), stream)
    plan = capi.load().sb_hash_aggregate_last_plan().decode()
    assert plan.startswith("rtc:"), plan


# ------------------------------------------------------------------------------------------------ 2. Partial buffers
@pytest.mark.parametrize("layout", ["none", "g33", "wide"])
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_partial_buffers_then_final(gpu, stream, tname, layout):
    """Partial output of two halves matches the reference's buffers bit for bit -- names (#sum, #count, #val, decimal
    #sum / #isEmpty), types (SUM(int8) bigint, MIN(decimal(7, 2)) decimal(7, 2), AVG double and bigint) and bits -- and Final
    over the partials concatenated in reverse order matches the Complete answer."""
    keys, aggs = A.key_names(layout), A.all_aggs(tname)
    t = A.value_table(tname, 20_011, layout, "nulls", seed=3)
    parts = []
    for half in (t.slice(0, 9000), t.slice(9000)):
        got = _check(half, keys, aggs, stream, mode="partial")
        want_types = [(f + sfx, ty) for f, _, _ in aggs for sfx, ty in A.buffer_types(f, tname)]
        assert [(f.name, f.type) for f in got.schema][len(keys):] == want_types
        parts.append(got)
    both = pa.concat_tables(parts[::-1])
    got = _agg(both, keys, aggs, stream, mode="final")
    A.assert_expected(got, A.expected(t, keys, aggs), len(keys))


# ------------------------------------------------------------------------------------------------ 3. AggregationState
def _cuts(t):
    n = t.num_rows
    return [t.slice(0, 0), t.slice(0, 1), t.slice(1, n // 2 - 1), t.slice(n // 2, 0), t.slice(n // 2)]


@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_batches_and_partial_merge(gpu, stream, tname):
    """execute_batches over cuts that include empty batches and a one-row batch (Complete); then a state fed the second half
    merges (sb_hash_agg_merge, PartialMerge) the Partial output of another state that saw the first half."""
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    aggs = A.all_aggs(tname)
    t = A.value_table(tname, 12_007, "g33", "nulls", seed=4)
    batches = [_batch(c, stream) for c in _cuts(t)]
    got = HashAggregateExec(["k"], _specs(aggs), LocalTableScanExec(batches[0])).execute_batches(batches, stream).to_arrow(stream)
    A.assert_expected(got, A.expected(t, ["k"], aggs), 1)

    half = t.num_rows // 2
    partial = HashAggregateExec(["k"], _specs(aggs), None, mode="partial")
    first = partial.execute_batches([_batch(t.slice(0, 1), stream), _batch(t.slice(1, half - 1), stream)], stream)
    second = _batch(t.slice(half), stream)
    state = partial.new_state(second)
    try:
        state.update(second, stream)
        state.merge(first, stream)
        merged = state.finish(stream)
    finally:
        state.close()
        first.close()
        second.close()
    A.assert_expected(merged.to_arrow(stream), A.expected(t, ["k"], aggs, mode="partial"), 1)
    got = HashAggregateExec(["k"], _specs(aggs), LocalTableScanExec(merged), mode="final").collect(stream)
    A.assert_expected(got, A.expected(t, ["k"], aggs), 1)


def test_sort_aggregate_is_the_same_operator(gpu, stream):
    from spark_b200.execution import SortAggregateExec
    for tname in ("dec7_2", "float32"):
        t = A.value_table(tname, 20_011, "g33", "nulls", seed=5)
        got = _agg(t, ["k"], A.all_aggs(tname), stream, cls=SortAggregateExec)
        A.assert_expected(got, A.expected(t, ["k"], A.all_aggs(tname)), 1)


# ------------------------------------------------------------------------------------------------ 4. Mixed plans through the decimal rewrite
def _mixed_table(n, seed):
    rng = np.random.default_rng(seed)
    base = A.value_table("dec7_2", n, "g33", "nulls", seed)
    cols = {"k": base.column("k"), "d": base.column("v")}
    for name, tname in (("d18", "dec18_0"), ("i8", "int8"), ("f32", "float32"), ("ts", "timestamp")):
        cols[name] = make_array(tname, A.ordinary_values(tname, n, rng), rng.random(n) >= 0.1)
    return pa.table(cols)


# Decimal SUM / AVG before, between and after other aggregates.  A Final / PartialMerge aggregate merges a decimal sum as four
# 32-bit limb sums and a count (five accumulator slots), so each plan holds two of them and stays within AGG_MAX_SLOTS in every mode.
MIXED = {
    "decimal_first": [("sum", "d", "s_d"), ("avg", "d18", "avg_d18"), ("min", "i8", "min_i8"), ("count", "f32", "n_f32")],
    "decimal_between": [("min", "i8", "min_i8"), ("sum", "d", "s_d"), ("count_star", None, "n"), ("avg", "d18", "avg_d18")],
    "decimal_last": [("sum", "i8", "s_i8"), ("max", "ts", "max_ts"), ("count", "f32", "n_f32"), ("sum", "d18", "s_d18")],
}


@pytest.mark.parametrize("order", list(MIXED))
@pytest.mark.parametrize("how", ["complete", "partial_final", "batches"])
@pytest.mark.parametrize("keys", [[], ["k"]])
def test_mixed_plan_through_the_decimal_rewrite(gpu, stream, keys, how, order):
    """Decimal SUM / AVG before, between and after MIN / MAX / COUNT / SUM over other types: hash_aggregate_decimals
    rebuilds the spec list (update modes) and plan_has_decimal_sums walks buffer positions (merge modes); every output must
    land in its own column with its own type."""
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    t = _mixed_table(30_011, 6)
    aggs = MIXED[order]
    if how == "complete":
        got = _agg(t, keys, aggs, stream)
    elif how == "partial_final":
        parts = []
        for half in (t.slice(0, 17_000), t.slice(17_000)):
            p = _agg(half, keys, aggs, stream, mode="partial")
            A.assert_expected(p, A.expected(half, keys, aggs, mode="partial"), len(keys))
            parts.append(p)
        got = _agg(pa.concat_tables(parts[::-1]), keys, aggs, stream, mode="final")
    else:
        batches = [_batch(c, stream) for c in _cuts(t)]
        got = HashAggregateExec(keys, _specs(aggs), LocalTableScanExec(batches[0])).execute_batches(batches, stream).to_arrow(stream)
    A.assert_expected(got, A.expected(t, keys, aggs), len(keys))


# ------------------------------------------------------------------------------------------------ 5. Slot budget
def test_sixteen_accumulator_slots_answer_seventeen_are_refused(gpu, stream):
    """AGG_MAX_SLOTS is 16.  MIN(c), MAX(c) and COUNT(c) of one nullable column take three slots -- the two extremes and one
    shared "seen" count (AggBuilder::add_slot merges equal slots) -- so five such columns take 15 and COUNT(*) the 16th.
    SUM(c0) adds a 17th (its own running sum; its "seen" count is c0's): refused with SB_ERR_UNSUPPORTED."""
    from spark_b200 import _capi as capi
    rng = np.random.default_rng(7)
    n = 5000
    cols = {"k": make_array("int32", rng.integers(0, 40, n).astype(np.int32))}
    aggs = [("count_star", None, "n")]
    for i in range(5):
        cols["c%d" % i] = make_array("int32", A.ordinary_values("int32", n, rng), rng.random(n) >= 0.1)
        aggs += [("min", "c%d" % i, "min%d" % i), ("max", "c%d" % i, "max%d" % i), ("count", "c%d" % i, "n%d" % i)]
    t = pa.table(cols)
    _check(t, ["k"], aggs, stream)
    with pytest.raises(capi.SparkB200Error) as e:
        _agg(t, ["k"], aggs + [("sum", "c0", "s0")], stream)
    assert e.value.code == 5


# ------------------------------------------------------------------------------------------------ 6. Empty global aggregate
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_empty_global_aggregate(gpu, stream, tname):
    """Zero rows, no keys: one row; COUNT is 0, SUM / AVG / MIN / MAX are NULL with their result types."""
    aggs = A.all_aggs(tname)
    t = pa.table({"v": make_array(tname, specials(tname)[:0])})
    got = _check(t, [], aggs, stream)
    assert got.num_rows == 1
    for f, _, name in aggs:
        assert got.schema.field(name).type == A.result_type(f, tname)
        assert got.column(name).to_pylist() == ([0] if f in ("count", "count_star") else [None])


# ------------------------------------------------------------------------------------------------ 7. Refusals
@pytest.mark.parametrize("func", ["sum", "avg", "min", "max", "count", "string_sum", "string_min"])
def test_unsupported_value_types_are_refused(gpu, stream, func):
    """decimal(38, 10) values (held in 128 bits) and string values are refused with SB_ERR_UNSUPPORTED, not answered."""
    import decimal as D
    from spark_b200 import _capi as capi
    rng = np.random.default_rng(8)
    n = 100
    if func.startswith("string_"):
        func = func[len("string_"):]
        v = pa.array(["x%d" % i for i in rng.integers(0, 50, n)])
    else:
        v = pa.array([D.Decimal(int(x)).scaleb(-10) for x in rng.integers(-10 ** 12, 10 ** 12, n)], pa.decimal128(38, 10))
    t = pa.table({"k": pa.array(rng.integers(0, 5, n).astype(np.int32)), "v": v})
    with pytest.raises(capi.SparkB200Error) as e:
        _agg(t, ["k"], [(func, "v", "r")], stream)
    assert e.value.code == 5
