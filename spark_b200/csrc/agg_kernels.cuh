// agg_kernels.cuh -- device side of HashAggregateExec (see aggregate.cu for the design notes and citations).
//
// The update kernels are templates over a *plan policy*:
//   DynPlan          metadata (types, operators, accumulator kinds, counts) is read from the kernel parameters;
//                    one binary serves every plan.
//   StaticPlan<&M>   metadata comes from a `__device__ const PlanMeta` table: after inlining, every descriptor loop has
//                    a constant trip count and unrolls, every type / mode / kind switch folds, and what is left per
//                    row is loads + arithmetic -- the same effect whole-stage codegen has on the reference's CPU path.
//                    The table and the instantiations are generated and compiled at run time (NVRTC, rtc.cu) when a
//                    plan first meets a large input; until then, and wherever NVRTC is unavailable, DynPlan runs (same
//                    code, same results).
#pragma once
#ifdef __CUDACC_RTC__
#include "device_helpers.cuh"   // run-time compilation (rtc.cu): device side only, headers come from the embedded copies
#else
#include "common.cuh"
#endif

namespace sb {

constexpr int AGG_THREADS = 128;
constexpr int AGG_DICT = 8;           // tier-1 dictionary entries per block
constexpr int AGG_MAX_SLOTS = 16;
constexpr int AGG_MAX_KEYS = 6;
constexpr int AGG_MAX_WORDS = 4;
constexpr int AGG_MAX_TERMS = 4;
constexpr int AGG_MAX_FACT = 3;
constexpr int AGG_MAX_COLS = 20;      // distinct input columns of one plan
constexpr int AGG_PROBE_LIMIT = 64;
constexpr uint64_t EMPTY_KEY = 0xFFFFFFFFFFFFFFFFull;

enum SlotKind { K_ADD_I64 = 0, K_ADD_F64 = 1, K_MIN_U64 = 2, K_MAX_U64 = 3 };
enum ValXform { X_NONE = 0, X_SIGNED = 1, X_DOUBLE = 2 };   // value -> order-preserving u64 for min/max
enum FactorMode { F_COL = 0, F_LIT_MINUS_COL = 1, F_LIT_PLUS_COL = 2, F_COL_MINUS_LIT = 3 };
enum SlotClass { CLS_GENERIC = 0, CLS_ONE = 1, CLS_F64_PRODUCT = 2 };   // ONE: count(*); F64_PRODUCT: non-null double factors
enum TermOp { T_EQ = 0, T_NE, T_LT, T_LE, T_GT, T_GE, T_NOTNULL };

// Everything about a plan that is not an address, a literal or a size.
struct PlanMeta {
  int32_t has_mask, nterms, single64, nkeys, nslots, pad;
  int32_t term_type[AGG_MAX_TERMS], term_op[AGG_MAX_TERMS], term_f64[AGG_MAX_TERMS], term_valid[AGG_MAX_TERMS];
  int32_t key_type[AGG_MAX_KEYS], key_bits[AGG_MAX_KEYS], key_shift[AGG_MAX_KEYS], key_nshift[AGG_MAX_KEYS], key_valid[AGG_MAX_KEYS];
  int32_t slot_kind[AGG_MAX_SLOTS], slot_nf[AGG_MAX_SLOTS], slot_one[AGG_MAX_SLOTS], slot_xform[AGG_MAX_SLOTS],
      slot_cls[AGG_MAX_SLOTS], slot_anyvalid[AGG_MAX_SLOTS];
  int32_t f_type[AGG_MAX_SLOTS][AGG_MAX_FACT], f_mode[AGG_MAX_SLOTS][AGG_MAX_FACT], f_valid[AGG_MAX_SLOTS][AGG_MAX_FACT];
  // every descriptor names its input by an index into AggArgs::col (distinct columns, numbered in order of first use:
  // mask, filter terms, keys, slot factors).  With a static plan two descriptors over the same column use the same
  // pointer expression, so the compiler merges their loads (Q1: 11 loads per row -> 7).
  int32_t ncols, mask_col;
  int32_t col_type[AGG_MAX_COLS];
  int32_t term_col[AGG_MAX_TERMS], key_col[AGG_MAX_KEYS], f_col[AGG_MAX_SLOTS][AGG_MAX_FACT];
};

struct ColRef {              // where one input buffer lives
  const void *data;          // HBM
  const uint8_t *valid;      // HBM validity bitmap or nullptr
};
struct KeyExtra {            // wide-key placement (multi-word keys only)
  int32_t word, null_word, hi_word, hi_shift;
};
struct AggArgs {
  PlanMeta meta;
  int64_t n;
  ColRef col[AGG_MAX_COLS];                      // distinct input columns (meta.*_col index into this)
  int64_t term_lit[AGG_MAX_TERMS];               // int64 value or double bits
  KeyExtra key_extra[AGG_MAX_KEYS];
  double fac_lit[AGG_MAX_SLOTS][AGG_MAX_FACT];
  int32_t nwords;
  uint64_t *tkeys;       // [nwords][cap + 2]   slot cap = NULL key, slot cap+1 = key equal to the EMPTY sentinel
  uint64_t *tacc;        // [nslots][cap + 2]
  int32_t *flags;        // [0] abort (table too small), [1] NULL-key slot used, [2] sentinel-key slot used,
                         // [6] / [7] the first / second dictionary kernel met a shape it should not handle (see gate)
  int64_t cap;
  // Automatic tier choice, no host round trip: the dictionary kernel runs with gate = 1; the first warp whose rows do not all
  // resolve in its block's dictionary (more than AGG_DICT groups, or NULL / sentinel keys) raises flags[6], every block stops at
  // its next tile boundary and leaves the number of tiles it finished in progress[block].  The shared-memory kernel is launched
  // right behind it with gate = 2: it returns at once when flags[6] is clear, otherwise it picks up the unfinished tiles.
  int32_t gate;          // 0: plain; 1: dictionary kernel, watch and yield; 2: shared-memory kernel, take over
  int32_t scap;          // shared-memory tier: table capacity (power of two)
  int32_t *progress;     // [dict_grid][warps]: tiles finished by every warp of the FIRST dictionary kernel's blocks
  int32_t *progress2;    // same shape, left by the second dictionary kernel (which works on the first one's tile geometry)
  int32_t dict_grid, dict_items;
  int32_t last_flag;     // index in flags of the yield flag of the LAST dictionary kernel of the chain (6 or 7)
  int32_t start_bypassed;   // shared-memory kernel: do not use the shared-memory table at all (tiny inputs: latency, not bandwidth)
  int32_t combine;       // shared-memory tier: combine same-entry rows of a warp before the atomics
};

struct DynPlan {
  static constexpr bool kStatic = false;
  static __device__ __forceinline__ const PlanMeta &meta(const AggArgs &a) { return a.meta; }
};
template <const PlanMeta *M>
struct StaticPlan {
  static constexpr bool kStatic = true;
  static __device__ __forceinline__ const PlanMeta &meta(const AggArgs &) { return *M; }
};
// descriptor loop: fully unrolled for a static plan (the bound folds to a constant), a plain loop otherwise
template <class P, class F>
__device__ __forceinline__ void plan_for(int n, F &&f) {
  if constexpr (P::kStatic) {
#pragma unroll
    for (int i = 0; i < n; i++) f(i);
  } else {
#pragma unroll 1
    for (int i = 0; i < n; i++) f(i);
  }
}

__device__ __forceinline__ uint64_t slot_identity(int kind) { return kind == K_MIN_U64 ? 0xFFFFFFFFFFFFFFFFull : 0ull; }

__device__ __forceinline__ uint64_t apply_op(int kind, uint64_t acc, uint64_t v) {
  switch (kind) {
    case K_ADD_I64: return acc + v;
    case K_ADD_F64: return (uint64_t)__double_as_longlong(__dadd_rn(__longlong_as_double((int64_t)acc), __longlong_as_double((int64_t)v)));
    case K_MIN_U64: return v < acc ? v : acc;
    default: return v > acc ? v : acc;
  }
}
__device__ __forceinline__ void global_op(int kind, uint64_t *addr, uint64_t v) {
  switch (kind) {
    case K_ADD_I64: atomicAdd((unsigned long long *)addr, (unsigned long long)v); break;
    case K_ADD_F64: atomicAdd((double *)addr, __longlong_as_double((int64_t)v)); break;
    case K_MIN_U64: atomicMin((unsigned long long *)addr, (unsigned long long)v); break;
    default: atomicMax((unsigned long long *)addr, (unsigned long long)v); break;
  }
}
__device__ __forceinline__ uint64_t mix64(uint64_t x) {   // slot choice only; not contractual
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// find-or-insert in the HBM table (single-word keys); returns slot index or -1 (abort: table too small).
// special: 0 regular key, 1 NULL key of a single 64-bit column, 2 a 64-bit key equal to the EMPTY sentinel.
__device__ __forceinline__ uint64_t table_home(const AggArgs &a, uint64_t key) { return mix64(key) & ((uint64_t)a.cap - 1); }
// continues a probe whose first word `cur` (the content of slot h) the caller has already fetched -- callers with several rows
// per thread issue all first-probe loads together, so the L2 round trips overlap instead of queueing behind one another
__device__ __forceinline__ int64_t table_slot_from(const AggArgs &a, uint64_t key, uint64_t h, uint64_t cur) {
  const uint64_t mask = (uint64_t)a.cap - 1;
  for (int step = 0; step < AGG_PROBE_LIMIT; step++) {
    if (cur == key) return (int64_t)h;
    if (cur == EMPTY_KEY) {
      uint64_t old = atomicCAS((unsigned long long *)&a.tkeys[h], (unsigned long long)EMPTY_KEY, (unsigned long long)key);
      if (old == EMPTY_KEY || old == key) return (int64_t)h;
    }
    h = (h + 1) & mask;
    cur = __ldcg(&a.tkeys[h]);
  }
  a.flags[0] = 1;
  return -1;
}
__device__ __forceinline__ int64_t table_slot(const AggArgs &a, uint64_t key, int special) {
  if (special == 1) { a.flags[1] = 1; return a.cap; }
  if (special == 2) { a.flags[2] = 1; return a.cap + 1; }
  const uint64_t h = table_home(a, key);
  return table_slot_from(a, key, h, __ldcg(&a.tkeys[h]));
}

// ---------------------------------------------------------------------------------------------------------
// Tile processing.  A thread owns ITEMS rows of a tile (row k = row0 + k*AGG_THREADS, coalesced per k); row0 is the absolute
// row and pointers are the column buffers in HBM.  FULL tiles use unclamped loads (LDG [base + k*stride] with immediate
// offsets, all ITEMS loads of a column in flight together).
// Every warp-uniform decision (column type, factor mode, accumulator kind) is taken OUTSIDE the unrolled row loop, and
// with a StaticPlan it is taken by the compiler.
// ---------------------------------------------------------------------------------------------------------
struct TileCtx {
  int64_t row0;
  int64_t last;           // clamp for partial tiles
};

// Column buffers are read-only HBM: loads go through ld.global.nc (__ldg), which tells the compiler they cannot alias the
// shared-memory accumulator stores, so it is free to hoist the loads of later slots above earlier accumulations and to
// merge repeated loads of the same column (a static plan's straight-line code then keeps a whole tile's loads in flight).
template <int ITEMS, bool FULL, typename T>
__device__ __forceinline__ void load_batch_as_i64(const void *__restrict__ data, const TileCtx &t, int64_t (&out)[ITEMS]) {
  const T *p = (const T *)data + t.row0;
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    if (FULL) out[k] = (int64_t)__ldg(p + k * AGG_THREADS);
    else {
      int64_t r = t.row0 + (int64_t)k * AGG_THREADS;
      out[k] = (int64_t)__ldg((const T *)data + (r < t.last ? r : t.last));
    }
  }
}
template <int ITEMS, bool FULL>
__device__ __forceinline__ void load_i64_batch(const void *__restrict__ data, int32_t type, const TileCtx &t, int64_t (&out)[ITEMS]) {
  switch (type) {
    case SB_BOOL: load_batch_as_i64<ITEMS, FULL, uint8_t>(data, t, out); break;
    case SB_INT8: load_batch_as_i64<ITEMS, FULL, int8_t>(data, t, out); break;
    case SB_INT16: load_batch_as_i64<ITEMS, FULL, int16_t>(data, t, out); break;
    case SB_INT32: case SB_DATE32: case SB_FLOAT32: load_batch_as_i64<ITEMS, FULL, int32_t>(data, t, out); break;
    default: load_batch_as_i64<ITEMS, FULL, int64_t>(data, t, out); break;
  }
}
template <int ITEMS, bool FULL>
__device__ __forceinline__ void load_f64_batch(const void *__restrict__ data, int32_t type, const TileCtx &t, double (&out)[ITEMS]) {
  if (type == SB_FLOAT64) {
    const double *p = (const double *)data + t.row0;
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      if (FULL) out[k] = __ldg(p + k * AGG_THREADS);
      else {
        int64_t r = t.row0 + (int64_t)k * AGG_THREADS;
        out[k] = __ldg((const double *)data + (r < t.last ? r : t.last));
      }
    }
  } else {
    int64_t x[ITEMS];
    load_i64_batch<ITEMS, FULL>(data, type, t, x);
    if (type == SB_FLOAT32) {
#pragma unroll
      for (int k = 0; k < ITEMS; k++) out[k] = (double)__int_as_float((int32_t)x[k]);
    } else {
#pragma unroll
      for (int k = 0; k < ITEMS; k++) out[k] = (double)x[k];
    }
  }
}
template <int ITEMS, bool FULL>
__device__ __forceinline__ void load_valid_batch(const uint8_t *__restrict__ valid, const TileCtx &t, bool (&out)[ITEMS]) {
  uint8_t b[ITEMS];
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    int64_t r = t.row0 + (int64_t)k * AGG_THREADS;
    if (!FULL) r = r < t.last ? r : t.last;
    b[k] = __ldg(valid + (r >> 3));
  }
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    int64_t r = t.row0 + (int64_t)k * AGG_THREADS;
    if (!FULL) r = r < t.last ? r : t.last;
    out[k] = (b[k] >> (r & 7)) & 1;
  }
}

// fused FilterExec: conjunction of column-vs-literal terms (a NULL comparison drops the row)
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void apply_filter_terms(const AggArgs &a, const TileCtx &t, bool (&keep)[ITEMS]) {
  const PlanMeta &m = P::meta(a);
  plan_for<P>(m.nterms, [&](int i) {
    if (m.term_valid[i]) {
      bool valid[ITEMS];
      load_valid_batch<ITEMS, FULL>(a.col[m.term_col[i]].valid, t, valid);
#pragma unroll
      for (int k = 0; k < ITEMS; k++) keep[k] = keep[k] && valid[k];
    }
    const int op = m.term_op[i];
    if (op == T_NOTNULL) return;
    int c[ITEMS];
    if (m.term_f64[i]) {
      double x[ITEMS];
      load_f64_batch<ITEMS, FULL>(a.col[m.term_col[i]].data, m.term_type[i], t, x);
      const double y = __longlong_as_double(a.term_lit[i]);
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {   // SQLOrderingUtil.compareDoubles
        bool xn = x[k] != x[k], yn = y != y;
        c[k] = x[k] == y ? 0 : (xn || yn) ? (int)xn - (int)yn : (x[k] < y ? -1 : 1);
      }
    } else {
      int64_t x[ITEMS];
      load_i64_batch<ITEMS, FULL>(a.col[m.term_col[i]].data, m.term_type[i], t, x);
      const int64_t lit = a.term_lit[i];
#pragma unroll
      for (int k = 0; k < ITEMS; k++) c[k] = x[k] == lit ? 0 : (x[k] < lit ? -1 : 1);
    }
    switch (op) {
#define SB_CMP(COND) _Pragma("unroll") for (int k = 0; k < ITEMS; k++) keep[k] = keep[k] && (COND);
      case T_EQ: SB_CMP(c[k] == 0) break;
      case T_NE: SB_CMP(c[k] != 0) break;
      case T_LT: SB_CMP(c[k] < 0) break;
      case T_LE: SB_CMP(c[k] <= 0) break;
      case T_GT: SB_CMP(c[k] > 0) break;
      default: SB_CMP(c[k] >= 0) break;
#undef SB_CMP
    }
  });
}

// value of factor f of slot s for the thread's rows: col | lit-col | lit+col | col-lit
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void factor_batch(const AggArgs &a, int s, int f, const TileCtx &t, double (&y)[ITEMS]) {
  const PlanMeta &m = P::meta(a);
  load_f64_batch<ITEMS, FULL>(a.col[m.f_col[s][f]].data, m.f_type[s][f], t, y);
  const int mode = m.f_mode[s][f];
  if (mode == F_COL) return;
  const double lit = a.fac_lit[s][f];
  switch (mode) {
    case F_LIT_MINUS_COL:
#pragma unroll
      for (int k = 0; k < ITEMS; k++) y[k] = __dsub_rn(lit, y[k]);
      break;
    case F_LIT_PLUS_COL:
#pragma unroll
      for (int k = 0; k < ITEMS; k++) y[k] = __dadd_rn(lit, y[k]);
      break;
    default:
#pragma unroll
      for (int k = 0; k < ITEMS; k++) y[k] = __dsub_rn(y[k], lit);
      break;
  }
}
// left-deep product of the slot's factors, evaluated in the reference's order ((f0*f1)*f2), no FMA contraction
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void product_batch(const AggArgs &a, int s, const TileCtx &t, double (&y)[ITEMS]) {
  const PlanMeta &m = P::meta(a);
  factor_batch<P, ITEMS, FULL>(a, s, 0, t, y);
  plan_for<P>(m.slot_nf[s] - 1, [&](int f1) {
    double z[ITEMS];
    factor_batch<P, ITEMS, FULL>(a, s, f1 + 1, t, z);
#pragma unroll
    for (int k = 0; k < ITEMS; k++) y[k] = __dmul_rn(y[k], z[k]);
  });
}

// 64-bit accumulator payload of slot s for the thread's rows
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void slot_values(const AggArgs &a, int s, const TileCtx &t, uint64_t (&v)[ITEMS]) {
  const PlanMeta &m = P::meta(a);
  const int kind = m.slot_kind[s], xform = m.slot_xform[s];
  if (m.slot_one[s]) {
#pragma unroll
    for (int k = 0; k < ITEMS; k++) v[k] = 1;
  } else if (kind == K_ADD_F64 || xform == X_DOUBLE) {
    double y[ITEMS];
    product_batch<P, ITEMS, FULL>(a, s, t, y);
    if (xform == X_DOUBLE) {   // order-preserving bits for min/max, NaN canonical (largest)
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {
        int64_t b = double_bits_canonical(y[k]);
        v[k] = (uint64_t)b ^ ((uint64_t)(b >> 63) | 0x8000000000000000ull);
      }
    } else {
#pragma unroll
      for (int k = 0; k < ITEMS; k++) v[k] = (uint64_t)__double_as_longlong(y[k]);
    }
  } else {
    int64_t x[ITEMS];
    load_i64_batch<ITEMS, FULL>(a.col[m.f_col[s][0]].data, m.f_type[s][0], t, x);
    const uint64_t flip = xform == X_SIGNED ? 0x8000000000000000ull : 0ull;
#pragma unroll
    for (int k = 0; k < ITEMS; k++) v[k] = (uint64_t)x[k] ^ flip;
  }
}

// rows whose inputs are NULL do not contribute (Sum.scala:113, Count.scala:94): ok[k] &= all factor columns valid
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void slot_input_valid(const AggArgs &a, int s, const TileCtx &t, bool (&ok)[ITEMS]) {
  const PlanMeta &m = P::meta(a);
  if (!m.slot_anyvalid[s]) return;
  plan_for<P>(m.slot_nf[s], [&](int f) {
    if (m.f_valid[s][f]) {
      bool valid[ITEMS];
      load_valid_batch<ITEMS, FULL>(a.col[m.f_col[s][f]].valid, t, valid);
#pragma unroll
      for (int k = 0; k < ITEMS; k++) ok[k] = ok[k] && valid[k];
    }
  });
}

// General accumulate: dst[k] >= 0: HBM table slot; doff[k] >= 0: offset of the row's group in the lane-private
// shared-memory accumulators (dictionary hit); both negative: row filtered out.
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void accumulate_slots(const AggArgs &a, const TileCtx &t, const int64_t (&dst)[ITEMS], const int (&doff)[ITEMS],
                                                 uint64_t *acc, int64_t stride) {
  const PlanMeta &m = P::meta(a);
  plan_for<P>(m.nslots, [&](int s) {
    uint64_t v[ITEMS];
    bool ok[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; k++) ok[k] = dst[k] >= 0 || doff[k] >= 0;
    slot_input_valid<P, ITEMS, FULL>(a, s, t, ok);
    slot_values<P, ITEMS, FULL>(a, s, t, v);
    uint64_t *sacc = acc + (size_t)s * AGG_THREADS;
    uint64_t *gacc = a.tacc + (int64_t)s * stride;
    switch (m.slot_kind[s]) {
#define SB_ACC(LOCAL, GLOBAL)                                          \
  _Pragma("unroll") for (int k = 0; k < ITEMS; k++) {                  \
    if (!ok[k]) continue;                                              \
    if (doff[k] >= 0) { uint64_t *p = sacc + doff[k]; LOCAL; }         \
    else { uint64_t *p = gacc + dst[k]; GLOBAL; }                      \
  }
      case K_ADD_F64:
        SB_ACC(*(double *)p = __dadd_rn(*(double *)p, __longlong_as_double((int64_t)v[k])),
               atomicAdd((double *)p, __longlong_as_double((int64_t)v[k])))
        break;
      case K_ADD_I64:
        SB_ACC(*p += v[k], atomicAdd((unsigned long long *)p, (unsigned long long)v[k]))
        break;
      case K_MIN_U64:
        SB_ACC(*p = v[k] < *p ? v[k] : *p, atomicMin((unsigned long long *)p, (unsigned long long)v[k]))
        break;
      default:
        SB_ACC(*p = v[k] > *p ? v[k] : *p, atomicMax((unsigned long long *)p, (unsigned long long)v[k]))
        break;
#undef SB_ACC
    }
  });
}

// Branch-free variant used when every kept row of the warp resolved to a dictionary entry: filtered rows and NULL
// inputs are steered to a "trash" accumulator group (index AGG_DICT), so the row loop is LDS + op + STS.
//
// Static plans take the two-phase form: phase 1 evaluates EVERY slot's payload for the thread's rows (no stores in
// between, so the compiler issues the loads of all referenced columns up front -- a whole tile in flight per warp);
// phase 2 walks rows outer / slots inner: for one row the slots' accumulators are acc + s*AGG_THREADS + doff[k] with s a
// compile-time constant, i.e. provably distinct addresses, so their LDS/op/STS chains overlap instead of forming one
// long read-after-write chain through shared memory.
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void accumulate_slots_dict(const AggArgs &a, const TileCtx &t, const int (&doff)[ITEMS], uint64_t *acc, int trash) {
  const PlanMeta &m = P::meta(a);
  if constexpr (P::kStatic) {
    uint64_t v[AGG_MAX_SLOTS][ITEMS];
    uint32_t nullbits[AGG_MAX_SLOTS];
    plan_for<P>(m.nslots, [&](int s) {
      nullbits[s] = 0;
      const int cls = m.slot_cls[s];
      if (cls == CLS_F64_PRODUCT) {
        double y[ITEMS];
        product_batch<P, ITEMS, FULL>(a, s, t, y);
#pragma unroll
        for (int k = 0; k < ITEMS; k++) v[s][k] = (uint64_t)__double_as_longlong(y[k]);
      } else if (cls == CLS_ONE) {
#pragma unroll
        for (int k = 0; k < ITEMS; k++) v[s][k] = 1;
      } else {
        bool ok[ITEMS];
#pragma unroll
        for (int k = 0; k < ITEMS; k++) ok[k] = true;
        slot_input_valid<P, ITEMS, FULL>(a, s, t, ok);
        slot_values<P, ITEMS, FULL>(a, s, t, v[s]);
#pragma unroll
        for (int k = 0; k < ITEMS; k++) nullbits[s] |= ok[k] ? 0u : (1u << k);
      }
    });
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      plan_for<P>(m.nslots, [&](int s) {
        uint64_t *p = acc + (size_t)s * AGG_THREADS + (((nullbits[s] >> k) & 1) ? trash : doff[k]);
        switch (m.slot_kind[s]) {
          case K_ADD_F64: *(double *)p = __dadd_rn(*(double *)p, __longlong_as_double((int64_t)v[s][k])); break;
          case K_ADD_I64: *p += v[s][k]; break;
          case K_MIN_U64: *p = v[s][k] < *p ? v[s][k] : *p; break;
          default: *p = v[s][k] > *p ? v[s][k] : *p; break;
        }
      });
    }
    return;
  }
  plan_for<P>(m.nslots, [&](int s) {
    uint64_t *sacc = acc + (size_t)s * AGG_THREADS;
    const int cls = m.slot_cls[s];
    if (cls == CLS_F64_PRODUCT) {
      double y[ITEMS];
      product_batch<P, ITEMS, FULL>(a, s, t, y);
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {
        double *p = (double *)(sacc + doff[k]);
        *p = __dadd_rn(*p, y[k]);
      }
    } else if (cls == CLS_ONE) {
#pragma unroll
      for (int k = 0; k < ITEMS; k++) sacc[doff[k]] += 1;
    } else {
      uint64_t v[ITEMS];
      bool ok[ITEMS];
#pragma unroll
      for (int k = 0; k < ITEMS; k++) ok[k] = true;
      slot_input_valid<P, ITEMS, FULL>(a, s, t, ok);
      slot_values<P, ITEMS, FULL>(a, s, t, v);
      switch (m.slot_kind[s]) {
#define SB_ACCD(EXPR) _Pragma("unroll") for (int k = 0; k < ITEMS; k++) { uint64_t *p = sacc + (ok[k] ? doff[k] : trash); EXPR; }
        case K_ADD_F64: SB_ACCD(*(double *)p = __dadd_rn(*(double *)p, __longlong_as_double((int64_t)v[k]))) break;
        case K_ADD_I64: SB_ACCD(*p += v[k]) break;
        case K_MIN_U64: SB_ACCD(*p = v[k] < *p ? v[k] : *p) break;
        default: SB_ACCD(*p = v[k] > *p ? v[k] : *p) break;
#undef SB_ACCD
      }
    }
  });
}

// Shared memory of the update kernels: uint64 dict_keys[D]; uint64 fill; uint64 acc[(D + 1) * nslots][AGG_THREADS]
// (last group = trash).
// keep / packed group key / special-slot class of the thread's rows
template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void tile_keys(const AggArgs &a, const TileCtx &t, bool (&keep)[ITEMS], uint64_t (&key)[ITEMS], int (&special)[ITEMS]) {
  const PlanMeta &m = P::meta(a);
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    keep[k] = FULL || t.row0 + (int64_t)k * AGG_THREADS <= t.last;
    key[k] = 0;
  }
  if (m.has_mask) {
    int64_t x[ITEMS];
    load_batch_as_i64<ITEMS, FULL, uint8_t>(a.col[m.mask_col].data, t, x);
#pragma unroll
    for (int k = 0; k < ITEMS; k++) keep[k] = keep[k] && x[k] != 0;
  }
  apply_filter_terms<P, ITEMS, FULL>(a, t, keep);
  // ---- group key packing --------------------------------------------------------------------------------
#pragma unroll
  for (int k = 0; k < ITEMS; k++) special[k] = 0;
  if (m.single64) {
    int64_t x[ITEMS];
    load_batch_as_i64<ITEMS, FULL, int64_t>(a.col[m.key_col[0]].data, t, x);      // raw 64-bit words
    if (m.key_type[0] == SB_FLOAT64) {   // NormalizeFloatingNumbers: -0.0 -> 0.0, NaN canonical
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {
        double d = __longlong_as_double(x[k]);
        x[k] = d == 0.0 ? 0ll : double_bits_canonical(d);
      }
    }
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      key[k] = (uint64_t)x[k];
      special[k] = key[k] == EMPTY_KEY ? 2 : 0;
    }
    if (m.key_valid[0]) {
      bool valid[ITEMS];
      load_valid_batch<ITEMS, FULL>(a.col[m.key_col[0]].valid, t, valid);
#pragma unroll
      for (int k = 0; k < ITEMS; k++) special[k] = valid[k] ? special[k] : 1;
    }
  } else {
    plan_for<P>(m.nkeys, [&](int i) {
      const int kt = m.key_type[i], bits = m.key_bits[i], shift = m.key_shift[i];
      int64_t x[ITEMS];
      load_i64_batch<ITEMS, FULL>(a.col[m.key_col[i]].data, kt, t, x);
      if (kt == SB_FLOAT32) {
#pragma unroll
        for (int k = 0; k < ITEMS; k++) {
          float f = __int_as_float((int32_t)x[k]);
          x[k] = f == 0.0f ? 0 : (int64_t)(uint32_t)float_bits_canonical(f);
        }
      }
      const uint64_t vmask = bits < 64 ? (1ull << bits) - 1 : ~0ull;
      if (m.key_valid[i]) {
        const int nshift = m.key_nshift[i];
        bool valid[ITEMS];
        load_valid_batch<ITEMS, FULL>(a.col[m.key_col[i]].valid, t, valid);
#pragma unroll
        for (int k = 0; k < ITEMS; k++) key[k] |= valid[k] ? ((uint64_t)x[k] & vmask) << shift : 1ull << nshift;
      } else {
#pragma unroll
        for (int k = 0; k < ITEMS; k++) key[k] |= ((uint64_t)x[k] & vmask) << shift;
      }
    });
  }
}

template <class P, int ITEMS, bool FULL, bool YIELD = false, int D = AGG_DICT>
__device__ __forceinline__ bool process_tile(const AggArgs &a, const TileCtx &t, uint64_t *dict_keys, uint64_t *acc, int tid, int64_t stride) {
  const PlanMeta &m = P::meta(a);
  const int ns = m.nslots;
  bool keep[ITEMS];
  uint64_t key[ITEMS];
  int special[ITEMS];
  tile_keys<P, ITEMS, FULL>(a, t, keep, key, special);
  // ---- where does each row accumulate? ---------------------------------------------------------------------
  int64_t dst[ITEMS];
  int doff[ITEMS];
  const int trash = D * ns * AGG_THREADS + tid;
  bool all_dict = true;
  // The dictionary's keys are compared in REGISTERS: D shared-memory loads per tile instead of a hashed probe loop per row.  A
  // row that matches none of the cached keys takes the slow path (linear probing with an atomicCAS claim, which also finds
  // entries other warps inserted since the snapshot) and refreshes the snapshot.
  constexpr bool SNAPSHOT = D <= 8;        // larger dictionaries (light plans only) are probed by hash: 2 x D registers is too many
  constexpr int DS = SNAPSHOT ? D : 1;
  uint64_t dk[DS];
  if constexpr (SNAPSHOT) {
#pragma unroll
    for (int i = 0; i < DS; i++) dk[i] = *(volatile uint64_t *)&dict_keys[i];
  }
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    dst[k] = -1;
    doff[k] = -1;
    if (!keep[k]) continue;
    if (YIELD && !all_dict) continue;   // this warp is going to yield: no point in resolving the rest of its rows
    int gid = -1;
    if (special[k] == 0) {
      if constexpr (SNAPSHOT) {
#pragma unroll
        for (int i = 0; i < DS; i++) gid = dk[i] == key[k] ? i : gid;
      }
      if (gid < 0) {
        constexpr int LOG_D = D == 4 ? 2 : (D == 8 ? 3 : (D == 16 ? 4 : 5));
        static_assert(D == 4 || D == 8 || D == 16 || D == 32, "dictionary sizes are powers of two");
        const uint32_t h0 = ((uint32_t)key[k] ^ (uint32_t)(key[k] >> 32)) * 0x9E3779B1u >> (32 - LOG_D);
        // a hash-probed dictionary gives up after 8 steps (inserts obey the same window, so lookups stay exact): near-full
        // tables would otherwise cost tens of probes per row -- with 32 keys in 32 entries the kernel ran 4x slower than the
        // shared-memory tier it is meant to beat
        constexpr int PROBES = D <= 8 ? D : 8;
#pragma unroll 1
        for (int i = 0; i < PROBES; i++) {
          const int g = (h0 + i) & (D - 1);
          uint64_t cur = *(volatile uint64_t *)&dict_keys[g];
          if (cur == EMPTY_KEY) {
            // a nearly full 32-entry dictionary is slower than the shared-memory tier: it stops at 20 keys
            if (!SNAPSHOT && *(volatile uint64_t *)&dict_keys[D] >= (uint64_t)(D * 5 / 8)) break;
            uint64_t old = atomicCAS((unsigned long long *)&dict_keys[g], (unsigned long long)EMPTY_KEY, (unsigned long long)key[k]);
            if (old == EMPTY_KEY && !SNAPSHOT) atomicAdd((unsigned long long *)&dict_keys[D], 1ull);
            cur = old == EMPTY_KEY ? key[k] : old;
          }
          if (cur == key[k]) { gid = g; break; }
        }
        if constexpr (SNAPSHOT) {
#pragma unroll
          for (int i = 0; i < DS; i++) dk[i] = *(volatile uint64_t *)&dict_keys[i];
        }
      }
    }
    if (gid >= 0) doff[k] = gid * ns * AGG_THREADS + tid;
    else {
      all_dict = false;
      if (!YIELD) dst[k] = table_slot(a, key[k], special[k]);
    }
  }
  if (YIELD) {   // watch-and-yield mode (AggArgs::gate == 1): a warp whose rows do not resolve in the dictionary leaves them untouched
    if (!__all_sync(0xffffffffu, all_dict)) return false;
#pragma unroll
    for (int k = 0; k < ITEMS; k++) doff[k] = doff[k] >= 0 ? doff[k] : trash;
    accumulate_slots_dict<P, ITEMS, FULL>(a, t, doff, acc, trash);
    return true;
  }
  if (__all_sync(0xffffffffu, all_dict)) {
#pragma unroll
    for (int k = 0; k < ITEMS; k++) doff[k] = doff[k] >= 0 ? doff[k] : trash;
    accumulate_slots_dict<P, ITEMS, FULL>(a, t, doff, acc, trash);
  } else {
    accumulate_slots<P, ITEMS, FULL>(a, t, dst, doff, acc, stride);
  }
  return true;
}

template <class P, int D = AGG_DICT>
__device__ __forceinline__ void dict_init(const AggArgs &a, uint64_t *dict_keys, uint64_t *acc, int tid) {
  const PlanMeta &m = P::meta(a);
  const int ns = m.nslots;
  if (tid < D) dict_keys[tid] = EMPTY_KEY;
  if (tid == 0) dict_keys[D] = 0;   // number of keys inserted (hash-probed dictionaries stop inserting at 5/8 load)
  for (int s = 0; s < ns; s++) {
    uint64_t id = slot_identity(m.slot_kind[s]);
    for (int g = 0; g <= D; g++) acc[(g * ns + s) * AGG_THREADS + tid] = id;
  }
}
// merge the block dictionary into the HBM table: one warp per GROUP -- one find-or-insert for the group, then a shuffle tree
// and one fire-and-forget RED per slot (a probe per (group, slot) pair made the kernel's tail a chain of L2 round trips)
template <class P, int D = AGG_DICT>
__device__ __forceinline__ void dict_merge(const AggArgs &a, const uint64_t *dict_keys, const uint64_t *acc, int tid, int64_t stride) {
  const PlanMeta &m = P::meta(a);
  const int ns = m.nslots;
  const int lane = tid & 31, warp = tid >> 5, nwarps = AGG_THREADS / 32;
  for (int g = warp; g < D; g += nwarps) {
    const uint64_t key = dict_keys[g];
    if (key == EMPTY_KEY) continue;
    int64_t slot = 0;
    if (lane == 0) slot = table_slot(a, key, 0);
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (slot < 0) continue;
    plan_for<P>(ns, [&](int s) {
      const int kind = m.slot_kind[s];
      const uint64_t *p = acc + (size_t)(g * ns + s) * AGG_THREADS;
      uint64_t v = slot_identity(kind);
#pragma unroll
      for (int i = 0; i < AGG_THREADS / 32; i++) v = apply_op(kind, v, p[lane + 32 * i]);
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) v = apply_op(kind, v, __shfl_xor_sync(0xffffffffu, v, d));
      if (lane == 0) global_op(kind, &a.tacc[(int64_t)s * stride + slot], v);
    });
  }
}

// L2 prefetch of the tile this block will process next (direct path): one prefetch.global.L2 per future load, issued before
// the current tile's compute, so the next tile's loads find their lines in L2 (~300 cycles) instead of HBM (~1000) and the
// 16 resident warps per SM need far fewer bytes in flight to keep HBM busy.  Costs no registers.
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
template <int ITEMS>
__device__ __forceinline__ void prefetch_col(const void *data, int32_t type, int64_t row0) {
  if (!data) return;
  const int w = type == SB_STRING ? 0 : (type == SB_BOOL || type == SB_INT8 ? 1 : type == SB_INT16 ? 2
                : (type == SB_INT32 || type == SB_FLOAT32 || type == SB_DATE32) ? 4 : 8);
  const uint8_t *p = (const uint8_t *)data + row0 * w;
#pragma unroll
  for (int k = 0; k < ITEMS; k++) prefetch_l2(p + (int64_t)k * AGG_THREADS * w);
}
template <class P, int ITEMS>
__device__ __forceinline__ void prefetch_tile(const AggArgs &a, int64_t row0) {
  const PlanMeta &m = P::meta(a);
  plan_for<P>(m.ncols, [&](int c) { prefetch_col<ITEMS>(a.col[c].data, m.col_type[c], row0); });
}

// ---- direct kernel: columns are read straight from HBM --------------------------------------------------------------
// MODE 0: plain (rows the dictionary cannot hold go to the HBM table).
// MODE 1: watch and yield -- the first kernel of the automatic chain: a warp whose rows do not all resolve in the D-entry
//         dictionary leaves them untouched, raises flags[6] and records its progress; everybody else stops at the next tile.
// MODE 2: take over and yield -- the second kernel of the chain (a larger dictionary, lower occupancy): returns at once unless
//         flags[6] is set, then walks the warp slices the first kernel left behind (same tile geometry), and yields in turn
//         (flags[7], progress2) to the shared-memory kernel.
// Lane-private accumulators cost D x slots x 8 bytes per thread, so the dictionary size sets the occupancy: Q1 (6 slots) keeps
// 28 warps per SM with D = 4 against 16 with D = 8 -- the 4-group query runs faster at the higher occupancy -- and a 5..8-group
// input costs one extra launch.
enum { AGG_MODE_PLAIN = 0, AGG_MODE_YIELD = 1, AGG_MODE_TAKEOVER = 2 };
template <class P, int ITEMS, bool PREFETCH = false, int MODE = AGG_MODE_PLAIN, int D = AGG_DICT>
__global__ void __launch_bounds__(AGG_THREADS) agg_update_kernel(const __grid_constant__ AggArgs a) {
  extern __shared__ __align__(128) uint64_t sm_direct[];
  uint64_t *dict_keys = sm_direct;
  uint64_t *acc = sm_direct + D + 1;   // [D] keys, one fill counter, accumulators
  const int tid = threadIdx.x;
  if (MODE == AGG_MODE_TAKEOVER && *(volatile int32_t *)&a.flags[6] == 0) return;   // the first kernel finished the job
  dict_init<P, D>(a, dict_keys, acc, tid);
  __syncthreads();
  constexpr int64_t TILE = (int64_t)AGG_THREADS * ITEMS;
  constexpr bool YIELD = MODE != AGG_MODE_PLAIN;
  const int64_t stride = a.cap + 2;
  volatile int32_t *yield_flag = &a.flags[MODE == AGG_MODE_TAKEOVER ? 7 : 6];
  // The abort / yield flags are sampled while a tile is being processed and acted on before the next one, so their L2 round trip
  // hides behind the tile's own loads.  Yielding is per WARP (no block barrier in the hot loop): a warp records how many tiles
  // it finished; the next kernel mirrors the tile geometry and picks up exactly the warp slices left behind.
  int32_t stop = 0;
  auto one_tile = [&](int64_t base, int64_t next) -> bool {   // false: this warp yields (the tile is untouched)
    stop = *(volatile int32_t *)a.flags;                       // another block found the table too small: give up early
    if (YIELD) stop |= *yield_flag;                            // somebody met rows this tier should not handle
    TileCtx t{base + tid, a.n - 1};
    if (PREFETCH && next + TILE <= a.n) prefetch_tile<P, ITEMS>(a, next + tid);
    if constexpr (YIELD) {
      const bool done = base + TILE <= a.n ? process_tile<P, ITEMS, true, true, D>(a, t, dict_keys, acc, tid, stride)
                                           : process_tile<P, ITEMS, false, true, D>(a, t, dict_keys, acc, tid, stride);
      if (!done) {
        *yield_flag = 1;
        return false;
      }
    } else if (base + TILE <= a.n) process_tile<P, ITEMS, true, false, D>(a, t, dict_keys, acc, tid, stride);
    else process_tile<P, ITEMS, false, false, D>(a, t, dict_keys, acc, tid, stride);
    return true;
  };
  if constexpr (MODE == AGG_MODE_TAKEOVER) {
    const int w = tid >> 5, lane = tid & 31;
    constexpr int NW = AGG_THREADS / 32;
    __shared__ int next_b;
    bool yielded = false;
    for (;;) {   // the first kernel's blocks are handed out dynamically (its grid is not a multiple of ours)
      if (tid == 0) next_b = atomicAdd(&a.flags[3], 1);
      __syncthreads();
      const int64_t b = next_b;
      __syncthreads();
      if (b >= a.dict_grid) break;
      int64_t j = a.progress[b * NW + w];   // this warp's slice of block b's tiles j, j + 1, ...
      if (!yielded) {
        for (;; j++) {
          const int64_t base = (b + j * a.dict_grid) * TILE;
          if (base >= a.n) break;
          if (stop || !one_tile(base, base + (int64_t)a.dict_grid * TILE)) {
            yielded = true;
            break;
          }
        }
      }
      if (lane == 0) a.progress2[b * NW + w] = (int32_t)j;
    }
  } else {
    int32_t tiles_done = 0;
    for (int64_t base = (int64_t)blockIdx.x * TILE; base < a.n && !stop; base += (int64_t)gridDim.x * TILE) {
      if (!one_tile(base, base + (int64_t)gridDim.x * TILE)) break;
      tiles_done++;
    }
    if (YIELD && (tid & 31) == 0) a.progress[blockIdx.x * (AGG_THREADS / 32) + (tid >> 5)] = tiles_done;
  }
  __syncthreads();
  dict_merge<P, D>(a, dict_keys, acc, tid, stride);
}

// ---- shared-memory tier: medium cardinality ----------------------------------------------------------------------------------
// Between "a handful of groups" (lane-private dictionary above) and "millions" (HBM table) sits the common GROUP BY over a
// dimension attribute: hundreds to a few thousand groups.  Sending every row to the HBM table then means tens of millions of
// atomics on a few thousand L2 lines (an order of magnitude slower than a handful of groups).  Here one 1024-thread block per SM keeps an
// open-addressing table in shared memory (keys + one accumulator array per slot, shared-memory atomics), and flushes it into
// the HBM table once at the end.  The table stops inserting at 75 % load; rows whose key is not resident take the HBM path,
// and when that becomes the norm (high cardinality) the block stops probing altogether.
// The block is eight 128-thread sub-blocks, each walking its own tiles with the tile geometry the loaders assume.
constexpr int AGGS_SUB = 8;
constexpr int AGGS_THREADS = AGG_THREADS * AGGS_SUB;
constexpr int AGGS_PROBES = 8;
enum { CTL_FILL = 0, CTL_BYPASS = 1, CTL_ROWS = 2, CTL_HITS = 3, CTL_SPECIAL = 4 /* and 5 */, CTL_WORDS = 8 };

__device__ __forceinline__ void shared_op(int kind, uint64_t *p, uint64_t v) {
  switch (kind) {
    case K_ADD_I64: {   // a 64-bit shared-memory add is a compare-and-swap loop; two native 32-bit adds with a carry are not
      uint32_t *w = (uint32_t *)p;
      const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
      const uint32_t old = atomicAdd(w, lo);
      const uint32_t carry = old + lo < old ? 1u : 0u;
      if (hi + carry) atomicAdd(w + 1, hi + carry);
      break;
    }
    case K_ADD_F64: atomicAdd((double *)p, __longlong_as_double((int64_t)v)); break;
    case K_MIN_U64: atomicMin((unsigned long long *)p, (unsigned long long)v); break;
    default: atomicMax((unsigned long long *)p, (unsigned long long)v); break;
  }
}

template <class P, int ITEMS, bool FULL>
__device__ __forceinline__ void process_tile_smem(const AggArgs &a, const TileCtx &t, uint64_t *skeys, uint64_t *sacc, uint32_t *sctl,
                                                  int64_t stride) {
  const PlanMeta &m = P::meta(a);
  bool keep[ITEMS];
  uint64_t key[ITEMS];
  int special[ITEMS];
  tile_keys<P, ITEMS, FULL>(a, t, keep, key, special);
  const uint32_t C = (uint32_t)a.scap, cmask = C - 1, fill_limit = C - (C >> 2);
  volatile uint32_t *vctl = sctl;
  // control words change under our feet: take one reading per warp so that warp-collective code below stays converged
  const bool bypass = __shfl_sync(0xffffffffu, vctl[CTL_BYPASS], 0) != 0;
  int64_t dst[ITEMS];
  int soff[ITEMS];
  uint32_t rows = 0, hits = 0;
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    dst[k] = -1;
    soff[k] = -1;
    if (!keep[k]) continue;
    rows++;
    if (special[k]) {   // NULL key / key equal to the EMPTY sentinel: two fixed entries behind the table
      soff[k] = (int)C + special[k] - 1;
      vctl[CTL_SPECIAL + special[k] - 1] = 1;
      hits++;
      continue;
    }
    if (!bypass) {
      uint32_t x = ((uint32_t)key[k] ^ (uint32_t)(key[k] >> 32)) * 0x9E3779B1u;
      uint32_t h = (x ^ (x >> 15)) & cmask;
#pragma unroll 1
      for (int p = 0; p < AGGS_PROBES; p++) {
        uint64_t cur = *(volatile uint64_t *)&skeys[h];
        if (cur == EMPTY_KEY && vctl[CTL_FILL] < fill_limit) {
          cur = atomicCAS((unsigned long long *)&skeys[h], (unsigned long long)EMPTY_KEY, (unsigned long long)key[k]);
          if (cur == EMPTY_KEY) {
            atomicAdd(&sctl[CTL_FILL], 1u);
            cur = key[k];
          }
        }
        if (cur == key[k]) {
          soff[k] = (int)h;
          break;
        }
        if (cur == EMPTY_KEY) break;   // table closed for inserts and the key is not resident
        h = (h + 1) & cmask;
      }
    }
    if (soff[k] >= 0) hits++;
  }
  {   // rows bound for the HBM table: every first probe in flight before the first one is looked at
    uint64_t home[ITEMS], cur[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      home[k] = 0;
      cur[k] = 0;
      if (keep[k] && soff[k] < 0) {
        home[k] = table_home(a, key[k]);
        cur[k] = __ldcg(&a.tkeys[home[k]]);
      }
    }
#pragma unroll
    for (int k = 0; k < ITEMS; k++)
      if (keep[k] && soff[k] < 0) dst[k] = table_slot_from(a, key[k], home[k], cur[k]);
  }
  // once the table is full, watch the hit rate: a block that mostly misses stops probing (high cardinality)
  if (!bypass && __shfl_sync(0xffffffffu, vctl[CTL_FILL], 0) >= fill_limit) {
    rows = __reduce_add_sync(0xffffffffu, rows);
    hits = __reduce_add_sync(0xffffffffu, hits);
    if ((threadIdx.x & 31) == 0) {
      uint32_t r = atomicAdd(&sctl[CTL_ROWS], rows) + rows, hh = atomicAdd(&sctl[CTL_HITS], hits) + hits;
      if (r >= 16384 && hh * 2 < r) vctl[CTL_BYPASS] = 1;
    }
  }
  // Rows of one warp that land on the same entry: with few distinct keys per warp every lane would fight for the same words
  // (a 64-bit shared-memory atomic is a compare-and-swap loop), so when some entry has 3+ takers the lanes first combine their
  // values through shuffles and only the lowest lane of every entry goes to memory.
  // Only the compare-and-swap kinds need this (double sums, min, max; int64 sums use native 32-bit adds), a.combine says
  // whether the plan has any.  MATCH is a slow instruction, so the check is rationed: every tile while the table holds few keys
  // (where crowding is the norm), every 8th tile otherwise (hot keys among many still get relief there, and a crowded
  // compare-and-swap is slow, not stuck).
  uint32_t grp[ITEMS];
  bool heavy = false;
  const bool check = a.combine && (__shfl_sync(0xffffffffu, vctl[CTL_FILL] < 256u, 0) || ((t.row0 >> 9) & 7) == 0);
  if (check) {
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      const uint32_t d = soff[k] >= 0 ? (uint32_t)soff[k] : 0x80000000u | (threadIdx.x & 31);   // HBM-bound rows are not combined
      grp[k] = __match_any_sync(0xffffffffu, d);
      heavy |= __popc(grp[k]) >= 3;
    }
    heavy = __any_sync(0xffffffffu, heavy);
  }
  const int lane = threadIdx.x & 31;
  plan_for<P>(m.nslots, [&](int s) {
    uint64_t v[ITEMS];
    bool ok[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; k++) ok[k] = dst[k] >= 0 || soff[k] >= 0;
    slot_input_valid<P, ITEMS, FULL>(a, s, t, ok);
    slot_values<P, ITEMS, FULL>(a, s, t, v);
    uint64_t *lacc = sacc + (size_t)s * (C + 2);
    uint64_t *gacc = a.tacc + (int64_t)s * stride;
    const int kind = m.slot_kind[s];
    if (heavy && kind != K_ADD_I64) {
      // every lane walks the OTHER members of its entry's group, lowest lane first; the trip count is the largest group of
      // the warp (uniform, so the shuffles stay convergent) -- a fixed 32-step loop cost 2500 thread-instructions per row
      const uint64_t ident = slot_identity(kind);
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {
        const uint64_t x = ok[k] ? v[k] : ident;
        uint32_t m = grp[k] & ~(1u << lane);
        const int trips = __reduce_max_sync(0xffffffffu, __popc(m));
        uint64_t acc = x;
#pragma unroll 1
        for (int t = 0; t < trips; t++) {
          const bool more = m != 0;
          const int src = more ? __ffs(m) - 1 : lane;
          m &= m - 1;
          const uint64_t o = __shfl_sync(0xffffffffu, x, src);
          if (more) acc = apply_op(kind, acc, o);
        }
        const bool leader = (grp[k] & lanemask_lt()) == 0;
        v[k] = acc;
        ok[k] = leader && (dst[k] >= 0 || soff[k] >= 0);
      }
    }
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      if (!ok[k]) continue;
      if (soff[k] >= 0) shared_op(kind, lacc + soff[k], v[k]);
      else global_op(kind, gacc + dst[k], v[k]);
    }
  });
}

template <class P, int ITEMS>
__global__ void __launch_bounds__(AGGS_THREADS) agg_update_smem_kernel(const __grid_constant__ AggArgs a) {
  extern __shared__ __align__(128) uint64_t sm_tab[];
  if (a.gate == 2 && *(volatile int32_t *)&a.flags[a.last_flag] == 0) return;   // the dictionary tiers finished the job
  const PlanMeta &m = P::meta(a);
  const int ns = m.nslots;
  const uint32_t C = (uint32_t)a.scap;
  uint64_t *skeys = sm_tab;                       // [C + 2]
  uint64_t *sacc = sm_tab + (C + 2);              // [ns][C + 2]
  uint32_t *sctl = (uint32_t *)(sacc + (size_t)ns * (C + 2));
  for (uint32_t i = threadIdx.x; i < C + 2; i += AGGS_THREADS) {
    skeys[i] = EMPTY_KEY;
    for (int s = 0; s < ns; s++) sacc[(size_t)s * (C + 2) + i] = slot_identity(m.slot_kind[s]);
  }
  if (threadIdx.x < CTL_WORDS) sctl[threadIdx.x] = (threadIdx.x == CTL_BYPASS && a.start_bypassed) ? 1u : 0u;
  __syncthreads();
  constexpr int64_t TILE = (int64_t)AGG_THREADS * ITEMS;
  const int64_t stride = a.cap + 2;
  const int tid = threadIdx.x & (AGG_THREADS - 1);
  const int64_t vb = (int64_t)blockIdx.x * AGGS_SUB + (threadIdx.x / AGG_THREADS), nvb = (int64_t)gridDim.x * AGGS_SUB;
  auto one_tile = [&](int64_t base) {
    TileCtx t{base + tid, a.n - 1};
    if (base + TILE <= a.n) process_tile_smem<P, ITEMS, true>(a, t, skeys, sacc, sctl, stride);
    else process_tile_smem<P, ITEMS, false>(a, t, skeys, sacc, sctl, stride);
  };
  if (a.gate == 2) {   // the tiles the dictionary kernels left behind (their tile = dict_items / ITEMS of ours)
    // every sub-block walks ALL dictionary tiles in its own strided order and skips, warp by warp, what is already done: the
    // work stays balanced whatever the dictionary kernels' grid was
    const int64_t dtile = (int64_t)AGG_THREADS * a.dict_items;
    const int64_t ndtiles = (a.n + dtile - 1) / dtile;
    const int w = tid >> 5;
    for (int64_t t = vb; t < ndtiles; t += nvb) {
      if (*(volatile int32_t *)a.flags) break;
      const int64_t b = t % a.dict_grid, j = t / a.dict_grid;
      if (j < a.progress2[b * (AGG_THREADS / 32) + w]) continue;
      const int64_t base0 = t * dtile;
      for (int64_t base = base0; base < base0 + dtile && base < a.n; base += TILE) one_tile(base);
    }
  } else {
    for (int64_t base = vb * TILE; base < a.n; base += nvb * TILE) {
      if (*(volatile int32_t *)a.flags) break;
      one_tile(base);
    }
  }
  __syncthreads();
  for (uint32_t h = threadIdx.x; h < C + 2; h += AGGS_THREADS) {
    int64_t slot;
    if (h < C) {
      const uint64_t key = skeys[h];
      if (key == EMPTY_KEY) continue;
      slot = table_slot(a, key, 0);
    } else {
      if (!sctl[CTL_SPECIAL + (h - C)]) continue;
      slot = table_slot(a, 0, (int)(h - C) + 1);
    }
    if (slot < 0) continue;
    for (int s = 0; s < ns; s++) global_op(m.slot_kind[s], &a.tacc[(int64_t)s * stride + slot], sacc[(size_t)s * (C + 2) + h]);
  }
}

// ---- wide grouping keys (> 63 bits, e.g. Q3's (l_orderkey, o_orderdate, o_shippriority)) -----------------------------
// Wait-free find-or-insert for multi-word keys.  Every key word carries at most 63 payload bits (bit 63 is 0), so no word
// of a real key equals EMPTY_KEY.  A thread claims the words of a slot in order with atomicCAS(EMPTY -> w[i]); a word
// already holding w[i] counts as claimed.  The first mismatch means the slot belongs to another key (probe on).  The key a
// slot ends up with is always some thread's full key: word i is set by the first thread whose words 0..i-1 matched.
// Nobody ever waits on anybody, so intra-warp divergence cannot deadlock.
template <int NW>
__device__ __forceinline__ int64_t table_slot_wide(const AggArgs &a, const uint64_t (&w)[NW]) {
  const int64_t stride = a.cap + 2;
  uint64_t mask = (uint64_t)a.cap - 1;
  uint64_t hh = 0;
#pragma unroll
  for (int i = 0; i < NW; i++) hh = mix64(hh ^ w[i]);
  uint64_t h = hh & mask;
  for (int step = 0; step < AGG_PROBE_LIMIT; step++) {
    bool match = true;
#pragma unroll
    for (int i = 0; i < NW; i++) {
      if (!match) break;
      uint64_t *p = &a.tkeys[(int64_t)i * stride + h];
      uint64_t cur = *(volatile uint64_t *)p;
      if (cur == EMPTY_KEY) {
        cur = atomicCAS((unsigned long long *)p, (unsigned long long)EMPTY_KEY, (unsigned long long)w[i]);
        if (cur == EMPTY_KEY) cur = w[i];
      }
      match = cur == w[i];
    }
    if (match) return (int64_t)h;
    h = (h + 1) & mask;
  }
  a.flags[0] = 1;
  return -1;
}

// keep / packed multi-word group key of the thread's rows (the wide-key counterpart of tile_keys)
template <int NW, int ITEMS>
__device__ __forceinline__ void tile_keys_wide(const AggArgs &a, const TileCtx &t, bool (&keep)[ITEMS], uint64_t (&key)[ITEMS][NW]) {
  using P = DynPlan;
  const PlanMeta &m = a.meta;
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    keep[k] = t.row0 + (int64_t)k * AGG_THREADS <= t.last;
#pragma unroll
    for (int i = 0; i < NW; i++) key[k][i] = 0;
  }
  if (m.has_mask) {
    int64_t x[ITEMS];
    load_batch_as_i64<ITEMS, false, uint8_t>(a.col[m.mask_col].data, t, x);
#pragma unroll
    for (int k = 0; k < ITEMS; k++) keep[k] = keep[k] && x[k] != 0;
  }
  apply_filter_terms<P, ITEMS, false>(a, t, keep);
  for (int i = 0; i < m.nkeys; i++) {
    const int kt = m.key_type[i], bits = m.key_bits[i], shift = m.key_shift[i];
    const KeyExtra ke = a.key_extra[i];
    int64_t x[ITEMS];
    bool valid[ITEMS];
    if (kt == SB_FLOAT64) load_batch_as_i64<ITEMS, false, int64_t>(a.col[m.key_col[i]].data, t, x);
    else load_i64_batch<ITEMS, false>(a.col[m.key_col[i]].data, kt, t, x);
    if (m.key_valid[i]) load_valid_batch<ITEMS, false>(a.col[m.key_col[i]].valid, t, valid);
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      if (m.key_valid[i] && !valid[k]) {
        const uint64_t nb = 1ull << m.key_nshift[i];
#pragma unroll
        for (int wi = 0; wi < NW; wi++)
          if (wi == ke.null_word) key[k][wi] |= nb;
        continue;
      }
      uint64_t v;
      if (kt == SB_FLOAT32) {
        float f = __int_as_float((int32_t)x[k]);
        v = f == 0.0f ? 0u : (uint32_t)float_bits_canonical(f);
      } else if (kt == SB_FLOAT64) {
        double d = __longlong_as_double(x[k]);
        v = d == 0.0 ? 0ull : (uint64_t)double_bits_canonical(d);
      } else {
        v = (uint64_t)x[k];
        if (bits < 64) v &= (1ull << bits) - 1;
      }
      if (bits == 64) {   // 63 payload bits per word: bit 63 lives elsewhere
        const uint64_t hi = (v >> 63) << ke.hi_shift;
#pragma unroll
        for (int wi = 0; wi < NW; wi++)
          if (wi == ke.hi_word) key[k][wi] |= hi;
        v &= 0x7FFFFFFFFFFFFFFFull;
      }
      v <<= shift;
#pragma unroll
      for (int wi = 0; wi < NW; wi++)
        if (wi == ke.word) key[k][wi] |= v;
    }
  }
}

template <int NW, int ITEMS>
__global__ void __launch_bounds__(AGG_THREADS) agg_update_wide_kernel(const __grid_constant__ AggArgs a) {
  using P = DynPlan;
  const int tid = threadIdx.x;
  constexpr int64_t TILE = (int64_t)AGG_THREADS * ITEMS;
  const int64_t stride = a.cap + 2;
  for (int64_t base = (int64_t)blockIdx.x * TILE; base < a.n; base += (int64_t)gridDim.x * TILE) {
    if (*(volatile int32_t *)a.flags) break;
    TileCtx t{base + tid, a.n - 1};
    bool keep[ITEMS];
    uint64_t key[ITEMS][NW];
    tile_keys_wide<NW, ITEMS>(a, t, keep, key);
    int64_t dst[ITEMS];
    int doff[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; k++) {
      doff[k] = -1;
      dst[k] = keep[k] ? table_slot_wide<NW>(a, key[k]) : -1;
    }
    accumulate_slots<P, ITEMS, false>(a, t, dst, doff, nullptr, stride);
  }
}

}  // namespace sb
