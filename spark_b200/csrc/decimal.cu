// decimal.cu -- SUM and AVG over DecimalType columns.
//
// Reference semantics (sql/catalyst/.../expressions/aggregate/Sum.scala:80-178, Average.scala:80-135, non-ANSI):
//   Sum(decimal(p, s))     -> decimal(min(p + 10, 38), s); buffer = (sum, isEmpty); NULL for no non-NULL input, NULL on overflow of
//                             the result precision;
//   Average(decimal(p, s)) -> decimal(min(p + 4, 38), s + 4); buffer = (sum decimal(p + 10, s), count bigint); result =
//                             sum / count rounded HALF_UP (Decimal./ rounds to 39 fractional digits first, which cannot change
//                             the second rounding for a divisor below 2^63), NULL on overflow.
// A decimal(p <= 18) column is an int64 of unscaled values (SB_DECIMAL64); sums need up to 128 bits.  The hash-aggregate kernels
// accumulate 64-bit words, so a decimal sum is accumulated as LIMB sums: value = hi * 2^32 + lo with lo = the low 32 bits
// (unsigned) and hi = the rest (signed) -- each limb sum stays far inside int64 for 2^31 rows -- and recomposed in 128-bit
// arithmetic when the result is emitted.  Merging (Final / PartialMerge) does the same with the four 32-bit limbs of the 128-bit
// partial sums.  The rewrite happens here, around the fixed-width aggregate: temporary limb columns in, composed columns out;
// the kernels of agg_kernels.cuh are unchanged.
#include <vector>
#include "decimal.cuh"
#include "expr.cuh"
#include "moments.cuh"

namespace sb {

typedef __int128 i128;

static inline bool is_decimal(int32_t t) { return t == SB_DECIMAL64 || t == SB_DECIMAL128; }
static inline int dec_precision(const Column &c) {
  const int p = SB_DECIMAL_PRECISION(c.scale);
  return p > 0 ? p : (c.type == SB_DECIMAL64 ? 18 : 38);
}
static inline int32_t dec_type_for(int precision) { return precision <= 18 ? SB_DECIMAL64 : SB_DECIMAL128; }

__device__ __forceinline__ i128 pow10_i128(int e) {
  i128 r = 1;
  for (int i = 0; i < e; i++) r *= 10;
  return r;
}
__device__ __forceinline__ i128 load_dec(const void *data, int32_t type, int64_t i) {
  if (type == SB_DECIMAL64) return (i128)((const int64_t *)data)[i];
  const uint64_t lo = ((const uint64_t *)data)[2 * i], hi = ((const uint64_t *)data)[2 * i + 1];
  return (i128)(((unsigned __int128)hi << 64) | lo);
}
__device__ __forceinline__ void store_dec(void *data, int32_t type, int64_t i, i128 v) {
  if (type == SB_DECIMAL64) {
    ((int64_t *)data)[i] = (int64_t)v;
    return;
  }
  ((uint64_t *)data)[2 * i] = (uint64_t)(unsigned __int128)v;
  ((uint64_t *)data)[2 * i + 1] = (uint64_t)((unsigned __int128)v >> 64);
}

// value -> limbs.  nlimbs = 2: (low 32 bits, value >> 32); nlimbs = 4: three unsigned 32-bit limbs and the signed top one.
// NULL rows contribute zeros; nonempty[i] = 1 for a non-NULL row (update modes count those) or = the row's own count column
__global__ void split_limbs_kernel(const void *__restrict__ data, const uint8_t *__restrict__ valid, int32_t type, int64_t n, int nlimbs,
                                   int64_t *__restrict__ l0, int64_t *__restrict__ l1, int64_t *__restrict__ l2, int64_t *__restrict__ l3) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const i128 v = bit_valid(valid, i) ? load_dec(data, type, i) : (i128)0;
  if (nlimbs == 2) {
    l0[i] = (int64_t)((uint64_t)v & 0xFFFFFFFFull);
    l1[i] = (int64_t)(v >> 32);
    return;
  }
  const unsigned __int128 u = (unsigned __int128)v;
  l0[i] = (int64_t)((uint64_t)u & 0xFFFFFFFFull);
  l1[i] = (int64_t)((uint64_t)(u >> 32) & 0xFFFFFFFFull);
  l2[i] = (int64_t)((uint64_t)(u >> 64) & 0xFFFFFFFFull);
  l3[i] = (int64_t)(int32_t)(uint32_t)(u >> 96);
}
// isEmpty (bool) -> 1 for "this partial sum has seen a value"
__global__ void nonempty_kernel(const uint8_t *__restrict__ is_empty, const uint8_t *__restrict__ valid, int64_t n, int64_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = bit_valid(valid, i) && !is_empty[i] ? 1 : 0;
}

struct LimbCols {
  const int64_t *l[4];
  const uint8_t *lv[4];   // validity of the limb sums (a group whose inputs were all NULL has NULL sums: read as 0)
  const int64_t *count;
  const uint8_t *count_valid;
  int nlimbs;
};
__device__ __forceinline__ i128 compose(const LimbCols &c, int64_t g) {
  i128 v = 0;
  for (int k = c.nlimbs - 1; k >= 0; k--) {
    const int64_t x = bit_valid(c.lv[k], g) ? c.l[k][g] : 0;
    v = v * ((i128)1 << 32) + (i128)x;   // wraps like the reference's BigDecimal would not, but an overflow is caught below
  }
  return v;
}
// what: 0 = sum buffer (value; 0 when empty), 1 = sum result (NULL when empty or beyond the precision), 2 = average result
__global__ void compose_kernel(LimbCols c, int64_t ngroups, int what, int precision, int in_scale_shift, int32_t out_type, void *__restrict__ out,
                               uint32_t *__restrict__ out_valid, uint8_t *__restrict__ is_empty_out, int64_t *__restrict__ count_out) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = g < ngroups;
  bool valid = false;
  if (in) {
    const int64_t cnt = bit_valid(c.count_valid, g) ? c.count[g] : 0;
    i128 v = compose(c, g);
    const i128 bound = pow10_i128(precision);
    if (what == 0) {
      valid = true;
      if (is_empty_out) is_empty_out[g] = cnt == 0;
      if (count_out) count_out[g] = cnt;
      if (cnt == 0) v = 0;
    } else if (what == 1) {
      valid = cnt > 0 && v < bound && v > -bound;
      if (!valid) v = 0;
    } else {
      if (cnt > 0) {   // round_half_up(sum * 10^4 / count) at scale s + 4
        const bool neg = v < 0;
        unsigned __int128 num = (unsigned __int128)(neg ? -v : v) * (unsigned __int128)pow10_i128(in_scale_shift);
        const unsigned __int128 den = (unsigned __int128)cnt;
        unsigned __int128 q = num / den;
        const unsigned __int128 rem = num % den;
        if (rem * 2 >= den) q += 1;
        v = neg ? -(i128)q : (i128)q;
        valid = v < bound && v > -bound;
      }
      if (!valid) v = 0;
    }
    store_dec(out, out_type, g, v);
  }
  if (out_valid) {
    const uint32_t w = __ballot_sync(0xffffffffu, in && valid);
    if ((threadIdx.x & 31) == 0 && g - (g & 31) < ngroups) out_valid[g >> 5] = w;
  }
}

static inline unsigned dblocks(int64_t n) { return (unsigned)((n + 255) / 256); }

struct DecAgg {
  bool decimal = false;
  bool avg = false;
  int in_precision = 0, in_scale = 0;   // of the aggregated column (update) or p of the ORIGINAL column recovered from the buffer (merge)
  int first_spec = 0, nspecs = 0;       // where its rewritten specs sit
};

static bool update_decimal_input(const sb_table *in, const sb_agg_spec &sp, int *col) {
  if (sp.func != SB_AGG_SUM && sp.func != SB_AGG_AVG) return false;
  int c;
  if (!expr_is_column(sp.input, &c) || c < 0 || c >= (int)in->cols.size()) return false;
  if (!is_decimal(in->cols[c].type)) return false;
  *col = c;
  return true;
}

bool plan_has_decimal_sums(const sb_table *in, const sb_agg_plan *plan) {
  if (!in || !plan) return false;
  const bool merge = plan->mode == SB_AGG_MODE_FINAL || plan->mode == SB_AGG_MODE_PARTIAL_MERGE;
  int pos = plan->nkeys;
  for (int i = 0; i < plan->naggs; i++) {
    const sb_agg_spec &sp = plan->aggs[i];
    if (!merge) {
      int c;
      if (update_decimal_input(in, sp, &c)) return true;
      continue;
    }
    if (pos >= (int)in->cols.size()) return false;
    const bool dec = (sp.func == SB_AGG_SUM || sp.func == SB_AGG_AVG) && is_decimal(in->cols[pos].type);
    if (dec) return true;
    pos += agg_buffer_width(sp.func);
  }
  return false;
}

void hash_aggregate_decimals(const sb_table *in, const sb_agg_plan *plan, cudaStream_t st, AggregateFn run, sb_table **out) {
  const bool merge = plan->mode == SB_AGG_MODE_FINAL || plan->mode == SB_AGG_MODE_PARTIAL_MERGE;
  const bool emit_buffers = plan->mode == SB_AGG_MODE_PARTIAL || plan->mode == SB_AGG_MODE_PARTIAL_MERGE;
  const int64_t n = in->nrows;
  // ---- the view the fixed-width aggregate sees, and the rewritten specs -------------------------------------------------------
  sb_table *view = table_new(n);
  struct Guard { sb_table *t; ~Guard() { if (t) table_free(t); } } gview{view};
  std::vector<sb_agg_spec> specs;
  std::vector<sb_expr_node> nodes;   // one COL node per rewritten update-mode spec (stable storage: reserved below)
  nodes.reserve((size_t)plan->naggs * 8 + 8);
  std::vector<DecAgg> info(plan->naggs);
  auto temp_i64 = [&]() {
    Column c = column_alloc(SB_INT64, 0, n, false, st);
    view->cols.push_back(c);
    return (int64_t *)c.data->ptr;
  };
  auto col_spec = [&](int func, int col) {
    sb_agg_spec s;
    memset(&s, 0, sizeof(s));
    s.func = func;
    nodes.push_back(sb_expr_node{SB_OP_COL, SB_VT_I64, col, 0, {0}});
    s.input.nodes = &nodes.back();
    s.input.n = 1;
    s.input.out_type = SB_INT64;
    return s;
  };
  if (!merge) {
    for (auto &c : in->cols) view->cols.push_back(column_share(c));
    for (int i = 0; i < plan->naggs; i++) {
      const sb_agg_spec &sp = plan->aggs[i];
      int c;
      if (!update_decimal_input(in, sp, &c)) {
        info[i].first_spec = (int)specs.size();
        info[i].nspecs = 1;
        specs.push_back(sp);
        continue;
      }
      const Column &src = in->cols[c];
      if (src.type != SB_DECIMAL64) fail(SB_ERR_UNSUPPORTED, "SUM / AVG over a decimal(p > 18) input column is not implemented");
      info[i].decimal = true;
      info[i].avg = sp.func == SB_AGG_AVG;
      info[i].in_precision = dec_precision(src);
      info[i].in_scale = SB_DECIMAL_SCALE(src.scale);
      info[i].first_spec = (int)specs.size();
      info[i].nspecs = 3;
      const int base = (int)view->cols.size();
      int64_t *lo = temp_i64(), *hi = temp_i64();
      if (n > 0) {
        split_limbs_kernel<<<dblocks(n), 256, 0, st>>>(src.d(), src.v(), src.type, n, 2, lo, hi, nullptr, nullptr);
        SB_LAUNCH_CHECK();
      }
      specs.push_back(col_spec(SB_AGG_SUM, base));
      specs.push_back(col_spec(SB_AGG_SUM, base + 1));
      sb_agg_spec cnt = sp;            // COUNT(column): the non-NULL rows
      cnt.func = SB_AGG_COUNT;
      specs.push_back(cnt);
    }
  } else {
    SB_REQUIRE(plan->nkeys <= (int)in->cols.size(), "Final aggregate: fewer input columns than keys");
    for (int k = 0; k < plan->nkeys; k++) view->cols.push_back(column_share(in->cols[k]));
    int pos = plan->nkeys;
    for (int i = 0; i < plan->naggs; i++) {
      const sb_agg_spec &sp = plan->aggs[i];
      const int nbuf = agg_buffer_width(sp.func);
      SB_REQUIRE(pos < (int)in->cols.size(), "Final aggregate expects buffer column %d but the input has %zu columns", pos, in->cols.size());
      const bool dec = (sp.func == SB_AGG_SUM || sp.func == SB_AGG_AVG) && is_decimal(in->cols[pos].type);
      info[i].first_spec = (int)specs.size();
      if (!dec) {
        for (int b = 0; b < nbuf; b++) {
          SB_REQUIRE(pos + b < (int)in->cols.size(), "Final aggregate: missing buffer column %d", pos + b);
          view->cols.push_back(column_share(in->cols[pos + b]));
        }
        pos += nbuf;
        info[i].nspecs = 1;
        specs.push_back(sp);
        continue;
      }
      // decimal buffers: (sum decimal(p + 10, s), isEmpty bool) for SUM, (sum, count bigint) for AVG
      SB_REQUIRE(pos + 1 < (int)in->cols.size(), "Final aggregate: a decimal sum buffer is (sum, isEmpty | count)");
      const Column &sum = in->cols[pos], &second = in->cols[pos + 1];
      info[i].decimal = true;
      info[i].avg = sp.func == SB_AGG_AVG;
      info[i].in_precision = dec_precision(sum) - 10 > 0 ? dec_precision(sum) - 10 : 1;   // p of the aggregated column (capped sums: see emit)
      info[i].in_scale = SB_DECIMAL_SCALE(sum.scale);
      info[i].nspecs = 5;
      int64_t *l[4];
      for (int k = 0; k < 4; k++) l[k] = temp_i64();
      int64_t *ne = temp_i64();
      if (n > 0) {
        split_limbs_kernel<<<dblocks(n), 256, 0, st>>>(sum.d(), sum.v(), sum.type, n, 4, l[0], l[1], l[2], l[3]);
        SB_LAUNCH_CHECK();
        if (info[i].avg) {
          SB_REQUIRE(second.type == SB_INT64, "avg buffer count must be int64");
          SB_CUDA(cudaMemcpyAsync(ne, second.d(), (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
        } else {
          SB_REQUIRE(second.type == SB_BOOL, "decimal sum buffer: the second column is isEmpty (boolean)");
          nonempty_kernel<<<dblocks(n), 256, 0, st>>>((const uint8_t *)second.d(), second.v(), n, ne);
          SB_LAUNCH_CHECK();
        }
      }
      for (int k = 0; k < 5; k++) {
        sb_agg_spec s;
        memset(&s, 0, sizeof(s));
        s.func = SB_AGG_SUM;
        specs.push_back(s);
      }
      pos += 2;
    }
  }
  std::vector<int32_t> key_cols(plan->nkeys > 0 ? plan->nkeys : 1);
  for (int k = 0; k < plan->nkeys; k++) key_cols[k] = merge ? k : plan->key_cols[k];
  if (merge)
    for (int k = 0; k < plan->nkeys; k++) SB_REQUIRE(plan->key_cols[k] == k, "Final aggregate: the keys are the first columns of the Partial layout");
  sb_agg_plan p2 = *plan;
  p2.key_cols = key_cols.data();
  p2.naggs = (int32_t)specs.size();
  p2.aggs = specs.data();
  sb_table *res = nullptr;
  run(view, &p2, st, &res);
  struct Guard2 { sb_table *t; ~Guard2() { if (t) table_free(t); } } gres{res};

  // ---- compose: keys ++ per aggregate its buffers / result --------------------------------------------------------------------
  const int64_t g = res->nrows;
  sb_table *t = table_new(g);
  try {
    for (int k = 0; k < plan->nkeys; k++) t->cols.push_back(column_share(res->cols[k]));
    // output position of rewritten spec j inside `res`: one result column, or in a buffer-emitting mode the spec's buffer columns
    std::vector<int> spec_col(specs.size() + 1);
    int at = plan->nkeys;
    for (size_t j = 0; j < specs.size(); j++) {
      spec_col[j] = at;
      at += emit_buffers ? agg_buffer_width(specs[j].func) : 1;
    }
    spec_col[specs.size()] = at;
    SB_REQUIRE(at == (int)res->cols.size(), "internal: aggregate result has %zu columns, expected %d", res->cols.size(), at);
    for (int i = 0; i < plan->naggs; i++) {
      const DecAgg &d = info[i];
      if (!d.decimal) {
        for (int cidx = spec_col[d.first_spec]; cidx < spec_col[d.first_spec + 1]; cidx++) t->cols.push_back(column_share(res->cols[cidx]));
        continue;
      }
      LimbCols lc;
      memset(&lc, 0, sizeof(lc));
      lc.nlimbs = d.nspecs - 1;
      for (int k = 0; k < lc.nlimbs; k++) {
        const Column &c = res->cols[spec_col[d.first_spec + k]];
        lc.l[k] = (const int64_t *)c.d();
        lc.lv[k] = c.v();
      }
      const Column &cc = res->cols[spec_col[d.first_spec + lc.nlimbs]];
      lc.count = (const int64_t *)cc.d();
      lc.count_valid = cc.v();
      const int sum_prec = d.in_precision + 10 > 38 ? 38 : d.in_precision + 10;
      if (emit_buffers) {
        const int32_t ty = dec_type_for(sum_prec);
        Column sumc = column_alloc(ty, SB_DECIMAL_TYPE(sum_prec, d.in_scale), g, false, st);
        t->cols.push_back(sumc);
        Column second = column_alloc(d.avg ? SB_INT64 : SB_BOOL, 0, g, false, st);
        t->cols.push_back(second);
        if (g > 0) {
          compose_kernel<<<dblocks(g), 256, 0, st>>>(lc, g, 0, sum_prec, 0, ty, sumc.data->ptr, nullptr, d.avg ? nullptr : (uint8_t *)second.data->ptr,
                                                    d.avg ? (int64_t *)second.data->ptr : nullptr);
          SB_LAUNCH_CHECK();
        }
      } else if (!d.avg) {
        const int32_t ty = dec_type_for(sum_prec);
        Column r = column_alloc(ty, SB_DECIMAL_TYPE(sum_prec, d.in_scale), g, true, st);
        t->cols.push_back(r);
        if (g > 0) {
          compose_kernel<<<dblocks(g), 256, 0, st>>>(lc, g, 1, sum_prec, 0, ty, r.data->ptr, (uint32_t *)r.validity->ptr, nullptr, nullptr);
          SB_LAUNCH_CHECK();
        }
      } else {
        const int avg_prec = d.in_precision + 4 > 38 ? 38 : d.in_precision + 4;
        const int avg_scale = d.in_scale + 4;
        SB_REQUIRE(avg_scale <= 38 && d.in_precision + 14 <= 38, "AVG over decimal(%d, %d): the quotient does not fit 128 bits", d.in_precision, d.in_scale);
        const int32_t ty = dec_type_for(avg_prec);
        Column r = column_alloc(ty, SB_DECIMAL_TYPE(avg_prec, avg_scale), g, true, st);
        t->cols.push_back(r);
        if (g > 0) {
          compose_kernel<<<dblocks(g), 256, 0, st>>>(lc, g, 2, avg_prec, 4, ty, r.data->ptr, (uint32_t *)r.validity->ptr, nullptr, nullptr);
          SB_LAUNCH_CHECK();
        }
      }
    }
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
  SB_CUDA(cudaStreamSynchronize(st));   // `view`, `res` and the temporaries are released on return
}

}  // namespace sb
