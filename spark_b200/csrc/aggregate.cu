// aggregate.cu -- HashAggregateExec on the GPU, with the child FilterExec / ProjectExec fused in.
//
// Reference path replaced (citations relative to the reference tree, SQLX = sql/core/src/main/scala/
// org/apache/spark/sql/execution):
//   SQLX/aggregate/HashAggregateExec.scala:50 (doConsumeWithKeys :907-1335: per row project key ->
//   hash -> map probe/insert -> update buffer), UnsafeFixedWidthAggregationMap.java:124-181 over
//   BytesToBytesMap.java:604-643 (open addressing), buffer algebra Sum.scala:113-178,
//   Average.scala:80-135, Count.scala:94-105, Min/Max; modes AggUtils.scala:131-208;
//   FilterExec/ProjectExec SQLX/basicPhysicalOperators.scala:47,245 (fused by WholeStageCodegen there,
//   fused here by evaluating the predicate and the aggregate input expressions inside the update kernel).
//
// GPU design (HBM-bound; no tensor cores):
//   * one pass over the referenced input columns (coalesced loads, nothing materialised when the
//     predicate is a conjunction of column-vs-literal comparisons and every aggregate input is a
//     left-deep product of <= 3 factors of the form col | lit-col | lit+col | col-lit, which covers
//     TPC-H style price*(1-disc)*(1+tax) arithmetic; anything else is materialised first by expr.cu);
//   * group keys packed into one 64-bit word (fixed-width columns + null bits, or one raw 64-bit
//     column with reserved slots for NULL and for the EMPTY sentinel value);
//   * three tiers, picked on the device by a chain of kernels that yield to one another (agg_kernels.cuh):
//     tier 1: per-block dictionary of the first 4 / 8 (light plans: 32) distinct keys with LANE-PRIVATE
//     shared-memory accumulators (no atomics, no bank conflicts) and the keys compared in registers -- this is
//     what makes 4-group aggregates (Q1) run at memory speed; tier 2: per-SM open-addressing table in shared
//     memory (hundreds to thousands of groups); tier 3: open-addressing table in HBM (linear probing,
//     atomicCAS on the key word, RED on the accumulators);
//   * identical accumulator slots are de-duplicated (sum(x) and avg(x) share their sum; count(*) and the
//     counts of non-nullable averages share one counter).
// Floating SUM/AVG are order-dependent in the reference too (partials merge in fetch order); parity is
// 1e-6 relative for them, exact for keys/counts/integer sums/min/max.
#include <algorithm>
#include <math.h>
#include <stdlib.h>
#include <map>
#include <memory>
#include <thread>
#include "agg_kernels.cuh"
#include "expr.cuh"
#include "primitives.cuh"
#include "rtc.cuh"
#include "strings.cuh"
#include "decimal.cuh"
#include "moments.cuh"

namespace sb {

// ---- plan-specialised kernels, generated when a plan first runs ------------------------------------------------------
// Every update kernel is a template over a plan policy (agg_kernels.cuh).  The generic instantiation (DynPlan) is compiled
// ahead of time and serves any plan.  When a plan first meets an input large enough for it to matter, its PlanMeta is
// printed into a `__device__ const` table, the same templates are instantiated over StaticPlan<&table> by NVRTC (rtc.cu),
// and the resulting kernels are cached by the plan's bytes (process + disk) -- what whole-stage codegen + Janino do for the
// reference's CPU path.  Nothing in this file knows the shape of any particular query.
constexpr int ITEMS_DIRECT = 8;   // rows per thread per tile, direct path (1024-row tiles)

typedef const void *AggKernel;    // a __global__ symbol or a cudaKernel_t from a run-time compiled library
template <class K>
static AggKernel kptr(K k) { return (const void *)k; }
static void launch_agg(AggKernel k, int grid, int threads, size_t smem, cudaStream_t st, const AggArgs &a) {
  void *args[] = {(void *)&a};
  SB_CUDA(cudaLaunchKernel(k, dim3((unsigned)grid), dim3((unsigned)threads), args, smem, st));
}
constexpr int ITEMS_SMEM = 4;     // shared-memory tier: 512 threads x 4 rows
struct KernelChoice {
  AggKernel direct;                   // plain dictionary kernel (8 entries)
  int items_direct;
  std::string name;
  AggKernel smem = kptr(agg_update_smem_kernel<DynPlan, ITEMS_SMEM>);
  // the automatic chain: k1 watches and yields (dictionary of k1_dict entries, k1_items rows per thread), k2 (optional, 8
  // entries, same tile geometry) takes over and yields in turn, smem finishes
  AggKernel k1 = nullptr, k2 = nullptr;
  int k1_dict = 4, k1_items = ITEMS_DIRECT;
  AggKernel k1_wide = nullptr;        // 8-entry watch-and-yield kernel: the first level when 8 entries cost no occupancy ...
  AggKernel k2_big = nullptr;         // ... followed by a 32-entry (hash-probed) take-over kernel: light plans with 9..32 groups
  int k2_dict = 8;
};

static thread_local std::string g_last_plan_name;

// Plans that read many columns per row keep more loads in flight with 4 rows per thread (more resident warps); narrow plans
// (group by k, sum v) prefer 8.
static int chain_items(const PlanMeta &m) { return (m.ncols >= 5 || m.nslots >= 4) ? 4 : ITEMS_DIRECT; }

enum { NEED_K1 = 1, NEED_K2 = 2, NEED_K1W = 4, NEED_K2B = 8, NEED_DIRECT = 16, NEED_SMEM = 32, NEED_ALL = 63 };

// One NVRTC program per kernel (they compile concurrently, ~1.5 s each; a plan needs two or three of them).
static std::string plan_source(const PlanMeta &m) {
  std::string src = "#include \"agg_kernels.cuh\"\nnamespace sb {\n__device__ const PlanMeta kPlan = {";
  static_assert(sizeof(PlanMeta) % 4 == 0, "PlanMeta is a table of int32");
  const int32_t *w = (const int32_t *)&m;
  for (size_t i = 0; i < sizeof(PlanMeta) / 4; i++) {
    src += std::to_string(w[i]);
    src += i + 1 < sizeof(PlanMeta) / 4 ? "," : "";
  }
  src += "};\nusing RP = StaticPlan<&kPlan>;\n}\n";
  return src;
}
static std::string kernel_expr(int which, int items) {
  const std::string it = std::to_string(items);
  switch (which) {
    case NEED_K1: return "sb::agg_update_kernel<sb::RP, " + it + ", false, 1, 4>";     // watch and yield, 4 entries
    case NEED_K2: return "sb::agg_update_kernel<sb::RP, " + it + ", false, 2, 8>";     // take over, 8 entries
    case NEED_K1W: return "sb::agg_update_kernel<sb::RP, " + it + ", false, 1, 8>";    // watch and yield, 8 entries
    case NEED_K2B: return "sb::agg_update_kernel<sb::RP, " + it + ", false, 2, 32>";   // take over, 32 entries (hash probed)
    case NEED_DIRECT: return "sb::agg_update_kernel<sb::RP, 8, true, 0, 8>";           // plain (caller knows: <= 8 groups)
    default: return "sb::agg_update_smem_kernel<sb::RP, 4>";
  }
}
// compiles (or fetches from the cache) the kernels in `need`; out[i] = kernel of bit i or nullptr.  Returns false when any failed.
static bool specialise_kernels(const PlanMeta &m, int items, int need, bool load, const void *out[6], std::string *log, bool *all_cached) {
  const std::string src = plan_source(m);
  const std::string base((const char *)&m, sizeof(PlanMeta));
  const RtcProgram *progs[6] = {nullptr};
  std::vector<std::thread> workers;
  for (int i = 0; i < 6; i++) {
    if (!(need & (1 << i))) continue;
    workers.emplace_back([&, i] {
      const std::string expr = kernel_expr(1 << i, items);
      progs[i] = rtc_compile(base + "/" + expr + (load ? "" : "/check"), src, {expr}, load);
    });
  }
  for (auto &t : workers) t.join();
  bool ok = true;
  if (all_cached) *all_cached = true;
  for (int i = 0; i < 6; i++) {
    out[i] = nullptr;
    if (!(need & (1 << i))) continue;
    if (!progs[i]->ok) {
      ok = false;
      if (log) *log = progs[i]->log;
      continue;
    }
    if (load) out[i] = progs[i]->kernels[0];
    if (log && !load) *log += progs[i]->log + "; ";
    if (all_cached && !progs[i]->from_disk_cache) *all_cached = false;
  }
  return ok;
}

struct SpecialisedSet {
  const void *k[6];
  bool ok, from_disk;
};
static bool specialise(const PlanMeta &m, int64_t n, int need, KernelChoice &kc) {
  const Config &cfg = config();
  if (!cfg.agg_rtc || n < cfg.agg_rtc_min_rows) return false;
  const int items = chain_items(m);
  // per-call fast path: one map lookup keyed by the plan's bytes (building the source text and joining compiler threads
  // on every batch cost more than the Final aggregate of a 4-group query)
  static std::mutex mu;
  static std::map<std::string, SpecialisedSet> known;
  std::string key((const char *)&m, sizeof(PlanMeta));
  key.push_back((char)need);
  SpecialisedSet set;
  bool have = false;
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = known.find(key);
    if (it != known.end()) { set = it->second; have = true; }
  }
  if (!have) {
    std::string log;
    set.ok = specialise_kernels(m, items, need, true, set.k, &log, &set.from_disk);
    if (!set.ok && cfg.agg_verbose) fprintf(stderr, "[sb_hash_aggregate] run-time specialisation unavailable, generic kernels used: %s\n", log.c_str());
    std::lock_guard<std::mutex> lk(mu);
    known[key] = set;
  }
  if (!set.ok) return false;
  const void *const *k = set.k;
  const bool cached = set.from_disk;
  if (k[0]) kc.k1 = k[0];
  if (k[1]) kc.k2 = k[1];
  if (k[2]) kc.k1_wide = k[2];
  if (k[3]) kc.k2_big = k[3];
  if (k[4]) { kc.direct = k[4]; kc.items_direct = 8; }
  if (k[5]) kc.smem = k[5];
  kc.k1_items = items;     // k1 / k2 / k1_wide / k2_big share one tile geometry: all of the chain's members are in `need`
  char hex[32];
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < sizeof(PlanMeta); i++) { h ^= ((const unsigned char *)&m)[i]; h *= 1099511628211ull; }
  snprintf(hex, sizeof(hex), "%016llx", (unsigned long long)h);
  kc.name = std::string("rtc:") + hex + (cached ? "(disk)" : "");
  return true;
}

static KernelChoice choose_kernels(const PlanMeta &m, int64_t n, int need) {
  KernelChoice kc{kptr(agg_update_kernel<DynPlan, ITEMS_DIRECT>), ITEMS_DIRECT, "generic"};
  kc.k1 = kptr(agg_update_kernel<DynPlan, ITEMS_DIRECT, false, AGG_MODE_YIELD, 4>);
  kc.k2 = kptr(agg_update_kernel<DynPlan, ITEMS_DIRECT, false, AGG_MODE_TAKEOVER, 8>);
  kc.k1_wide = kptr(agg_update_kernel<DynPlan, ITEMS_DIRECT, false, AGG_MODE_YIELD, 8>);
  kc.k2_big = kptr(agg_update_kernel<DynPlan, ITEMS_DIRECT, false, AGG_MODE_TAKEOVER, 32>);
  kc.k1_dict = 4;
  kc.k1_items = ITEMS_DIRECT;
  specialise(m, n, need, kc);
  return kc;
}

__global__ void occupied_kernel(const uint64_t *__restrict__ tkeys, int64_t cap, const int32_t *__restrict__ flags,
                                uint8_t *__restrict__ occ) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cap) occ[i] = tkeys[i] != EMPTY_KEY;
  else if (i == cap) occ[i] = flags[1] != 0;
  else if (i == cap + 1) occ[i] = flags[2] != 0;
}

// ---- emit: one thread per output group -------------------------------------------------------
struct EmitKey {
  void *out;
  uint32_t *out_valid;
  int32_t type, bits, shift, null_shift, word, null_word, hi_word, hi_shift;
};
enum EmitOp { E_RAW = 0, E_SUM_NULLABLE, E_AVG, E_MINMAX };
struct EmitCol {
  void *out;
  uint32_t *out_valid;
  int32_t op;         // EmitOp
  int32_t out_type;   // SB_INT64 / SB_FLOAT64 / source type for min/max
  int32_t slot;       // main accumulator
  int32_t slot2;      // seen-count / avg count (or -1)
  int32_t xform;      // for min/max
  int32_t pad;
};
struct EmitArgs {
  int32_t nkeys, single64, ncols, nwords;
  EmitKey key[AGG_MAX_KEYS];
  EmitCol col[2 * AGG_MAX_SLOTS];
  const uint64_t *tkeys;
  const uint64_t *tacc;
  const int64_t *slot_ids;
  int64_t cap, ngroups;
};

__device__ __forceinline__ void store_typed(void *out, int32_t type, int64_t i, int64_t v) {
  switch (type) {
    case SB_BOOL: case SB_INT8: ((int8_t *)out)[i] = (int8_t)v; break;
    case SB_INT16: ((int16_t *)out)[i] = (int16_t)v; break;
    case SB_INT32: case SB_DATE32: case SB_FLOAT32: ((int32_t *)out)[i] = (int32_t)v; break;
    default: ((int64_t *)out)[i] = v; break;
  }
}

__global__ void __launch_bounds__(256) agg_emit_kernel(const __grid_constant__ EmitArgs e) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool in_range = r < e.ngroups;
  int64_t slot = in_range ? e.slot_ids[r] : 0;
  const int64_t stride = e.cap + 2;
#pragma unroll 1
  for (int k = 0; k < e.nkeys; k++) {
    const EmitKey &ek = e.key[k];
    bool valid = in_range;
    int64_t v = 0;
    if (in_range) {
      uint64_t key = e.tkeys[(int64_t)ek.word * stride + slot];
      if (e.single64) {
        if (slot == e.cap) valid = false;                       // NULL group key
        else if (slot == e.cap + 1) v = (int64_t)EMPTY_KEY;
        else v = (int64_t)key;
      } else {
        if (ek.null_shift >= 0 && ((e.tkeys[(int64_t)ek.null_word * stride + slot] >> ek.null_shift) & 1)) valid = false;
        else {
          uint64_t u = key >> ek.shift;
          if (ek.bits == 64 && e.nwords > 1)
            u = (u & 0x7FFFFFFFFFFFFFFFull) | (((e.tkeys[(int64_t)ek.hi_word * stride + slot] >> ek.hi_shift) & 1) << 63);
          if (ek.bits < 64) {
            u &= (1ull << ek.bits) - 1;
            // sign-extend integer types
            if (ek.type != SB_BOOL && ek.type != SB_FLOAT32 && (u >> (ek.bits - 1)) & 1) u |= ~((1ull << ek.bits) - 1);
          }
          v = (int64_t)u;
        }
      }
      store_typed(ek.out, ek.type, r, valid ? v : 0);
    }
    if (ek.out_valid) {
      uint32_t w = __ballot_sync(0xffffffffu, valid);
      if ((threadIdx.x & 31) == 0 && (r - (r & 31)) < e.ngroups) ek.out_valid[r >> 5] = w;
    }
  }
#pragma unroll 1
  for (int c = 0; c < e.ncols; c++) {
    const EmitCol &ec = e.col[c];
    bool valid = in_range;
    if (in_range) {
      uint64_t m = e.tacc[(int64_t)ec.slot * stride + slot];
      uint64_t m2 = ec.slot2 >= 0 ? e.tacc[(int64_t)ec.slot2 * stride + slot] : 1;
      int64_t v = (int64_t)m;
      switch (ec.op) {
        case E_SUM_NULLABLE: valid = m2 != 0; break;            // all-NULL group -> NULL (Sum.scala:180)
        case E_AVG: {                                           // Average.scala:109-127: count == 0 -> NULL
          valid = m2 != 0;
          double s = __longlong_as_double((int64_t)m);
          v = valid ? __double_as_longlong(__ddiv_rn(s, (double)(int64_t)m2)) : 0;
          break;
        }
        case E_MINMAX: {
          valid = m2 != 0;
          if (ec.xform == X_SIGNED) v = (int64_t)(m ^ 0x8000000000000000ull);
          else if (ec.xform == X_DOUBLE) {
            uint64_t b = (m >> 63) ? (m ^ 0x8000000000000000ull) : ~m;
            v = (int64_t)b;
            if (ec.out_type == SB_FLOAT32) v = (int64_t)__float_as_int((float)__longlong_as_double((int64_t)b));
          }
          break;
        }
        default: break;
      }
      store_typed(ec.out, ec.out_type, r, valid ? v : 0);
    }
    if (ec.out_valid) {
      uint32_t w = __ballot_sync(0xffffffffu, valid);
      if ((threadIdx.x & 31) == 0 && (r - (r & 31)) < e.ngroups) ec.out_valid[r >> 5] = w;
    }
  }
}

// ==============================================================================================
// host side: plan -> kernel arguments
// ==============================================================================================
struct ExprTree {   // tiny tree view of a postfix program
  int op, vtype, arg;
  int64_t lit;
  int l = -1, r = -1;
};
static int build_tree(const sb_expr &e, std::vector<ExprTree> &t) {
  std::vector<int> stack;
  for (int i = 0; i < e.n; i++) {
    ExprTree nd;
    nd.op = e.nodes[i].op;
    nd.vtype = e.nodes[i].vtype;
    nd.arg = e.nodes[i].arg;
    nd.lit = e.nodes[i].lit.i;
    switch (nd.op) {
      case SB_OP_COL: case SB_OP_LIT_I64: case SB_OP_LIT_F64: case SB_OP_LIT_NULL: break;
      case SB_OP_STR_EQ: case SB_OP_STR_LT: case SB_OP_STR_LE: case SB_OP_STR_GT: case SB_OP_STR_GE: case SB_OP_STR_IN:
      case SB_OP_STR_STARTS_WITH: case SB_OP_STR_ENDS_WITH: case SB_OP_STR_CONTAINS: case SB_OP_STR_LIKE: case SB_OP_STR_OCTET_LENGTH: case SB_OP_STR_CHAR_LENGTH: break;
      case SB_OP_NEG: case SB_OP_NOT: case SB_OP_ISNULL: case SB_OP_ISNOTNULL:
      case SB_OP_CAST_F64: case SB_OP_CAST_I64: case SB_OP_CAST_I32:
        nd.l = stack.back(); stack.pop_back(); break;
      default:
        nd.r = stack.back(); stack.pop_back();
        nd.l = stack.back(); stack.pop_back();
    }
    t.push_back(nd);
    stack.push_back((int)t.size() - 1);
  }
  return stack.back();
}

// host view of one accumulator slot before it is split into PlanMeta + AggArgs arrays
struct HostFactor {
  const void *data = nullptr;
  const uint8_t *valid = nullptr;
  int32_t type = 0, mode = F_COL;
  double lit = 0;
};
struct HostRef {
  const void *data = nullptr;
  const uint8_t *valid = nullptr;
  int32_t type = 0;
};
struct HostSlot {
  int32_t kind = 0, nf = 0, is_one = 0, xform = X_NONE;
  HostFactor f[AGG_MAX_FACT];
};

// A column whose validity buffer is present but known to hold no NULL (null_count == 0: what ColumnVector.hasNull() == false
// is to the reference's readers) is treated as non-nullable: no bitmap is read for it.
static const uint8_t *nulls_of(const Column &c) { return (c.validity && c.null_count != 0) ? c.v() : nullptr; }

static bool is_f64_col(const sb_table *in, const ExprTree &n) { return n.op == SB_OP_COL && in->cols[n.arg].type == SB_FLOAT64; }
static double lit_as_double(const ExprTree &n) {
  if (n.op == SB_OP_LIT_F64) { double d; memcpy(&d, &n.lit, 8); return d; }
  return (double)n.lit;
}
static bool is_lit(const ExprTree &n) { return n.op == SB_OP_LIT_F64 || n.op == SB_OP_LIT_I64; }

static bool match_factor(const sb_table *in, const std::vector<ExprTree> &t, int i, HostFactor &f) {
  const ExprTree &n = t[i];
  auto set_col = [&](const ExprTree &c) {
    const Column &col = in->cols[c.arg];
    f.data = col.d(); f.valid = nulls_of(col); f.type = col.type;
  };
  if (is_f64_col(in, n)) { set_col(n); f.mode = F_COL; f.lit = 0; return true; }
  if (n.vtype != SB_VT_F64) return false;
  if (n.op == SB_OP_SUB && is_lit(t[n.l]) && is_f64_col(in, t[n.r])) { set_col(t[n.r]); f.mode = F_LIT_MINUS_COL; f.lit = lit_as_double(t[n.l]); return true; }
  if (n.op == SB_OP_SUB && is_f64_col(in, t[n.l]) && is_lit(t[n.r])) { set_col(t[n.l]); f.mode = F_COL_MINUS_LIT; f.lit = lit_as_double(t[n.r]); return true; }
  if (n.op == SB_OP_ADD && is_lit(t[n.l]) && is_f64_col(in, t[n.r])) { set_col(t[n.r]); f.mode = F_LIT_PLUS_COL; f.lit = lit_as_double(t[n.l]); return true; }
  if (n.op == SB_OP_ADD && is_f64_col(in, t[n.l]) && is_lit(t[n.r])) { set_col(t[n.l]); f.mode = F_LIT_PLUS_COL; f.lit = lit_as_double(t[n.r]); return true; }
  return false;
}

// left-deep product of <= 3 factors, evaluated in the reference's order ((f0*f1)*f2)
static bool match_product(const sb_table *in, const sb_expr &e, HostSlot &s) {
  std::vector<ExprTree> t;
  int root = build_tree(e, t);
  int chain[AGG_MAX_FACT], rights[AGG_MAX_FACT];
  int nf = 0, nr = 0, cur = root;
  while (t[cur].op == SB_OP_MUL && t[cur].vtype == SB_VT_F64 && nr < AGG_MAX_FACT - 1) {   // Mul(Mul(a,b),c) -> [a,b,c]
    rights[nr++] = t[cur].r;
    cur = t[cur].l;
  }
  chain[nf++] = cur;
  for (int k = nr - 1; k >= 0; k--) chain[nf++] = rights[k];
  HostFactor f[AGG_MAX_FACT];
  for (int k = 0; k < nf; k++)
    if (!match_factor(in, t, chain[k], f[k])) return false;
  s.nf = nf;
  for (int k = 0; k < nf; k++) s.f[k] = f[k];
  return true;
}

static bool match_filter(const sb_table *in, const sb_expr &e, AggArgs &a, HostRef *term_refs) {
  std::vector<ExprTree> t;
  int root = build_tree(e, t);
  std::vector<int> work{root};
  PlanMeta &m = a.meta;
  m.nterms = 0;
  while (!work.empty()) {
    int i = work.back();
    work.pop_back();
    const ExprTree &n = t[i];
    if (n.op == SB_OP_AND) { work.push_back(n.l); work.push_back(n.r); continue; }
    if (m.nterms >= AGG_MAX_TERMS) return false;
    const int ti = m.nterms;
    auto set = [&](const Column &c, int op, int is_f64, int64_t lit) {
      term_refs[ti] = {c.d(), nulls_of(c), c.type};
      m.term_type[ti] = c.type; m.term_op[ti] = op; m.term_f64[ti] = is_f64; m.term_valid[ti] = nulls_of(c) != nullptr;
      a.term_lit[ti] = lit;
      m.nterms++;
    };
    if (n.op == SB_OP_ISNOTNULL && t[n.l].op == SB_OP_COL && in->cols[t[n.l].arg].type != SB_STRING) {
      set(in->cols[t[n.l].arg], T_NOTNULL, 0, 0);
      continue;
    }
    if (n.op < SB_OP_EQ || n.op > SB_OP_GE) return false;
    int op = n.op - SB_OP_EQ;   // T_EQ..T_GE share the order of SB_OP_EQ..SB_OP_GE
    const ExprTree *col = &t[n.l], *lit = &t[n.r];
    if (is_lit(*col) && lit->op == SB_OP_COL) {   // lit cmp col -> flip
      std::swap(col, lit);
      static const int flip[6] = {T_EQ, T_NE, T_GT, T_GE, T_LT, T_LE};
      op = flip[op];
    }
    if (col->op != SB_OP_COL || !is_lit(*lit)) return false;
    const Column &c = in->cols[col->arg];
    if (c.type == SB_STRING) return false;
    if (n.arg == SB_VT_F64) {
      if (c.type != SB_FLOAT64 && c.type != SB_FLOAT32) return false;
      double d = lit_as_double(*lit);
      int64_t bits;
      memcpy(&bits, &d, 8);
      set(c, op, 1, bits);
    } else {
      if (c.type == SB_FLOAT64 || c.type == SB_FLOAT32 || lit->op != SB_OP_LIT_I64) return false;
      set(c, op, 0, lit->lit);
    }
  }
  return true;
}

static bool same_slot(const HostSlot &x, const HostSlot &y) {
  if (x.kind != y.kind || x.nf != y.nf || x.is_one != y.is_one || x.xform != y.xform) return false;
  for (int k = 0; k < x.nf; k++) {
    const HostFactor &a = x.f[k], &b = y.f[k];
    if (a.data != b.data || a.valid != b.valid || a.type != b.type || a.mode != b.mode) return false;
    if (memcmp(&a.lit, &b.lit, 8) != 0) return false;
  }
  return true;
}

struct AggBuilder {
  const sb_table *in;
  cudaStream_t st;
  std::vector<HostSlot> slots;
  std::vector<Column> temps;   // materialised expression results, released at the end

  int add_slot(HostSlot s) {
    if (s.is_one) {   // count(x) over a column that can never be NULL == count(*): only nullable columns matter
      int k2 = 0;
      for (int k = 0; k < s.nf; k++)
        if (s.f[k].valid) s.f[k2++] = s.f[k];
      s.nf = k2;
      for (int k = 0; k < s.nf; k++) { s.f[k].mode = F_COL; s.f[k].lit = 0; s.f[k].data = nullptr; s.f[k].type = 0; }
      for (int k = s.nf; k < AGG_MAX_FACT; k++) s.f[k] = HostFactor();
    }
    for (size_t i = 0; i < slots.size(); i++)
      if (same_slot(slots[i], s)) return (int)i;
    if ((int)slots.size() >= AGG_MAX_SLOTS) fail(SB_ERR_UNSUPPORTED, "aggregate needs more than %d accumulator slots", AGG_MAX_SLOTS);
    slots.push_back(s);
    return (int)slots.size() - 1;
  }

  // value source for an aggregate input expression
  HostSlot source_for(const sb_expr &e, int32_t *src_type) {
    HostSlot s;
    int col;
    if (expr_is_column(e, &col)) {
      SB_REQUIRE(col >= 0 && col < (int)in->cols.size(), "aggregate input column %d out of range", col);
      const Column &c = in->cols[col];
      if (c.type == SB_STRING) fail(SB_ERR_UNSUPPORTED, "aggregates over string columns are not supported");
      if (c.type == SB_DECIMAL128) fail(SB_ERR_UNSUPPORTED, "MIN / MAX / COUNT over decimal(p > 18) columns are not supported");
      s.nf = 1;
      s.f[0].data = c.d(); s.f[0].valid = nulls_of(c); s.f[0].type = c.type; s.f[0].mode = F_COL;
      *src_type = c.type;
      return s;
    }
    expr_validate(in, e);
    if (e.nodes[e.n - 1].vtype == SB_VT_F64 && match_product(in, e, s)) {
      *src_type = SB_FLOAT64;
      return s;
    }
    Column tmp = eval_projection(in, e, nullptr, in->nrows, st);   // general path: materialise
    temps.push_back(tmp);
    s.nf = 1;
    s.f[0].data = tmp.d(); s.f[0].valid = nulls_of(tmp); s.f[0].type = tmp.type; s.f[0].mode = F_COL;
    *src_type = tmp.type;
    return s;
  }
};

static bool is_float_type(int32_t t) { return t == SB_FLOAT32 || t == SB_FLOAT64; }

constexpr int OUT_MOMENT = -1;   // OutPlan::op of a column moments_run writes (csrc/moments.cu)
struct OutPlan {   // one output column
  int op, out_type, slot, slot2, xform;
  bool nullable;
  int32_t scale = 0;   // decimals: the source column's (precision, scale) for MIN / MAX
};

static int64_t next_pow2(int64_t x) {
  int64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

static void hash_aggregate_fixed(const sb_table *in, const sb_agg_plan *plan, cudaStream_t st, sb_table **out) {
  SB_REQUIRE(in && plan && out, "null argument");
  SB_REQUIRE(plan->mode >= SB_AGG_MODE_PARTIAL && plan->mode <= SB_AGG_MODE_PARTIAL_MERGE, "bad aggregate mode %d", plan->mode);
  SB_REQUIRE(plan->nkeys >= 0 && plan->naggs >= 0, "bad plan");
  const int64_t n = in->nrows;
  AggBuilder b;
  b.in = in;
  b.st = st;
  static thread_local AggArgs args_storage;
  AggArgs &a = args_storage;
  memset(&a, 0, sizeof(a));
  PlanMeta &m = a.meta;
  a.n = n;
  // distinct input columns, numbered in order of first use (mask, filter terms, keys, slot factors)
  auto col_index = [&](const void *data, const uint8_t *valid, int32_t type) -> int {
    for (int i = 0; i < m.ncols; i++)
      if (a.col[i].data == data && a.col[i].valid == valid && m.col_type[i] == type) return i;
    if (m.ncols >= AGG_MAX_COLS) fail(SB_ERR_UNSUPPORTED, "aggregate references more than %d distinct columns", AGG_MAX_COLS);
    a.col[m.ncols].data = data;
    a.col[m.ncols].valid = valid;
    m.col_type[m.ncols] = type;
    return m.ncols++;
  };
  std::vector<OutPlan> outs;
  std::vector<MomentInput> mom_in;
  std::vector<MomentOut> mom_out;
  std::vector<int> mom_first_out;   // index in `outs` of each moment aggregate's first column
  HostRef mask_ref, term_refs[AGG_MAX_TERMS], key_refs[AGG_MAX_KEYS];
  void *mask_ptr = nullptr;

  struct Cleanup {
    AggBuilder &b;
    void *&mask;
    cudaStream_t st;
    ~Cleanup() {
      for (auto &c : b.temps) column_release(c);
      if (mask) cudaFreeAsync(mask, st);
    }
  } cleanup{b, mask_ptr, st};

  // ---- keys --------------------------------------------------------------------------------
  SB_REQUIRE(plan->nkeys <= AGG_MAX_KEYS, "at most %d grouping keys are supported (got %d)", AGG_MAX_KEYS, plan->nkeys);
  m.nkeys = plan->nkeys;
  int total_bits = 0;
  for (int k = 0; k < plan->nkeys; k++) {
    int ci = plan->key_cols[k];
    SB_REQUIRE(ci >= 0 && ci < (int)in->cols.size(), "key column %d out of range", ci);
    const Column &c = in->cols[ci];
    SB_REQUIRE(c.type != SB_STRING, "string grouping keys reach the kernels as dictionary codes");
    if (c.type == SB_DECIMAL128) fail(SB_ERR_UNSUPPORTED, "decimal(p > 18) grouping keys are not supported");
    key_refs[k] = {c.d(), nulls_of(c), c.type};
    m.key_type[k] = c.type;
    m.key_bits[k] = type_width(c.type) * 8;
    m.key_valid[k] = nulls_of(c) != nullptr;
    m.key_nshift[k] = -1;
    total_bits += m.key_bits[k] + (m.key_valid[k] ? 1 : 0);
  }
  a.nwords = 1;
  if (plan->nkeys == 1 && m.key_bits[0] == 64) {
    m.single64 = 1;
  } else if (total_bits <= 63) {
    int pos = 0;
    for (int k = 0; k < plan->nkeys; k++) {
      m.key_shift[k] = pos;
      pos += m.key_bits[k];
      if (m.key_valid[k]) m.key_nshift[k] = pos++;
    }
  } else {
    // wide key: 63 payload bits per word (bit 63 stays 0 so a word never equals the EMPTY sentinel).  Value fields
    // first (a field never straddles words; a 64-bit field stores its low 63 bits and parks bit 63 with the flags),
    // then bit-63 spill bits and null flags in the free bits.
    int used[AGG_MAX_WORDS + 1] = {0};
    int nw = 0;
    auto place = [&](int nbits, int &word, int &shift) {
      int w = 0;
      while (w < AGG_MAX_WORDS && used[w] + nbits > 63) w++;
      if (w >= AGG_MAX_WORDS) fail(SB_ERR_UNSUPPORTED, "grouping keys do not fit in %d 63-bit words", AGG_MAX_WORDS);
      word = w;
      shift = used[w];
      used[w] += nbits;
      if (w + 1 > nw) nw = w + 1;
    };
    for (int k = 0; k < plan->nkeys; k++) {
      int word, shift;
      place(m.key_bits[k] == 64 ? 63 : m.key_bits[k], word, shift);
      a.key_extra[k].word = word;
      m.key_shift[k] = shift;
    }
    for (int k = 0; k < plan->nkeys; k++) {
      if (m.key_bits[k] == 64) {
        int word, shift;
        place(1, word, shift);
        a.key_extra[k].hi_word = word;
        a.key_extra[k].hi_shift = shift;
      }
      if (m.key_valid[k]) {
        int word, shift;
        place(1, word, shift);
        a.key_extra[k].null_word = word;
        m.key_nshift[k] = shift;
      }
    }
    a.nwords = nw < 2 ? 2 : nw;
  }

  // ---- fused filter ---------------------------------------------------------------------------
  if (plan->filter) {
    expr_validate(in, *plan->filter);
    if (!match_filter(in, *plan->filter, a, term_refs)) {
      m.nterms = 0;
      memset(m.term_type, 0, sizeof(m.term_type)); memset(m.term_op, 0, sizeof(m.term_op));
      memset(m.term_f64, 0, sizeof(m.term_f64)); memset(m.term_valid, 0, sizeof(m.term_valid));
      for (auto &r : term_refs) r = HostRef();
      memset(a.term_lit, 0, sizeof(a.term_lit));
      SB_CUDA(cudaMallocAsync(&mask_ptr, (size_t)n + 16, st));
      eval_predicate(in, *plan->filter, (uint8_t *)mask_ptr, st);
      mask_ref = {mask_ptr, nullptr, SB_INT8};
      m.has_mask = 1;
    }
  }

  // ---- aggregates -> accumulator slots + output plan -------------------------------------------
  // AggUtils.scala:131-208: Partial / PartialMerge emit buffers, Final / PartialMerge read buffers positionally
  const bool final_mode = plan->mode == SB_AGG_MODE_FINAL || plan->mode == SB_AGG_MODE_PARTIAL_MERGE;
  const bool emit_buffers = plan->mode == SB_AGG_MODE_PARTIAL || plan->mode == SB_AGG_MODE_PARTIAL_MERGE;
  int next_buf_col = plan->nkeys;   // Final: buffers follow the keys positionally
  for (int i = 0; i < plan->naggs; i++) {
    const sb_agg_spec &sp = plan->aggs[i];
    auto buffer_source = [&](int col) {
      SB_REQUIRE(col < (int)in->cols.size(), "Final aggregate expects buffer column %d but the input has %zu columns", col, in->cols.size());
      const Column &c = in->cols[col];
      HostSlot s;
      s.nf = 1;
      s.f[0].data = c.d(); s.f[0].valid = nulls_of(c); s.f[0].type = c.type; s.f[0].mode = F_COL;
      return s;
    };
    switch (sp.func) {
      case SB_AGG_SUM: {
        int32_t src_type;
        HostSlot s = final_mode ? buffer_source(next_buf_col) : b.source_for(sp.input, &src_type);
        if (final_mode) { src_type = in->cols[next_buf_col].type; next_buf_col++; }
        // Sum(decimal(p, s)) is decimal(p + 10, s) with an isEmpty flag and overflow -> NULL (Sum.scala:80-135): not an int64 sum
        if (src_type == SB_DECIMAL64) fail(SB_ERR_UNSUPPORTED, "SUM over a DECIMAL column is not implemented on the GPU path (needs decimal(p + 10, s) accumulation)");
        bool f64 = is_float_type(src_type) || s.nf > 1 || s.f[0].mode != F_COL;
        s.kind = f64 ? K_ADD_F64 : K_ADD_I64;
        // a global aggregate (no keys) over zero rows yields NULL, so it always tracks "seen"
        bool nullable = plan->nkeys == 0;
        for (int k = 0; k < s.nf; k++) nullable |= s.f[k].valid != nullptr;
        int main = b.add_slot(s);
        int seen = -1;
        if (nullable) {
          HostSlot c = s;
          c.kind = K_ADD_I64; c.is_one = 1;
          seen = b.add_slot(c);
        }
        outs.push_back({nullable ? E_SUM_NULLABLE : E_RAW, f64 ? SB_FLOAT64 : SB_INT64, main, seen, X_NONE, nullable});
        break;
      }
      case SB_AGG_AVG: {
        int sum_slot, cnt_slot;
        if (final_mode) {
          HostSlot s = buffer_source(next_buf_col); s.kind = K_ADD_F64;
          SB_REQUIRE(in->cols[next_buf_col].type == SB_FLOAT64, "avg buffer sum must be float64");
          HostSlot c = buffer_source(next_buf_col + 1); c.kind = K_ADD_I64;
          SB_REQUIRE(in->cols[next_buf_col + 1].type == SB_INT64, "avg buffer count must be int64");
          next_buf_col += 2;
          sum_slot = b.add_slot(s);
          cnt_slot = b.add_slot(c);
        } else {
          int32_t src_type;
          HostSlot s = b.source_for(sp.input, &src_type);
          // Average(decimal(p, s)) is decimal(p + 4, s + 4) (Average.scala:80-135): dividing the unscaled sum would be off by 10^s
          if (src_type == SB_DECIMAL64) fail(SB_ERR_UNSUPPORTED, "AVG over a DECIMAL column is not implemented on the GPU path");
          s.kind = K_ADD_F64;
          sum_slot = b.add_slot(s);
          HostSlot c = s;
          c.kind = K_ADD_I64; c.is_one = 1;
          cnt_slot = b.add_slot(c);
        }
        if (emit_buffers) {
          outs.push_back({E_RAW, SB_FLOAT64, sum_slot, -1, X_NONE, false});
          outs.push_back({E_RAW, SB_INT64, cnt_slot, -1, X_NONE, false});
        } else {
          outs.push_back({E_AVG, SB_FLOAT64, sum_slot, cnt_slot, X_NONE, true});
        }
        break;
      }
      case SB_AGG_COUNT: case SB_AGG_COUNT_STAR: {
        HostSlot s;
        if (final_mode) {
          s = buffer_source(next_buf_col);
          SB_REQUIRE(in->cols[next_buf_col].type == SB_INT64, "count buffer must be int64");
          next_buf_col++;
          s.kind = K_ADD_I64;
        } else if (sp.func == SB_AGG_COUNT) {
          int32_t src_type;
          s = b.source_for(sp.input, &src_type);
          s.kind = K_ADD_I64; s.is_one = 1;
        } else {
          s.kind = K_ADD_I64; s.is_one = 1; s.nf = 0;
        }
        outs.push_back({E_RAW, SB_INT64, b.add_slot(s), -1, X_NONE, false});
        break;
      }
      case SB_AGG_MIN: case SB_AGG_MAX: {
        int32_t src_type;
        HostSlot s = final_mode ? buffer_source(next_buf_col) : b.source_for(sp.input, &src_type);
        int32_t src_scale = 0;
        if (final_mode) { src_type = in->cols[next_buf_col].type; src_scale = in->cols[next_buf_col].scale; next_buf_col++; }
        else {
          int sc;
          if (expr_is_column(sp.input, &sc) && sc >= 0 && sc < (int)in->cols.size()) src_scale = in->cols[sc].scale;
        }
        if (s.nf != 1 || s.f[0].mode != F_COL) src_type = SB_FLOAT64;   // computed double expression
        s.kind = sp.func == SB_AGG_MIN ? K_MIN_U64 : K_MAX_U64;
        s.xform = is_float_type(src_type) ? X_DOUBLE : X_SIGNED;
        int main = b.add_slot(s);
        HostSlot c = s;
        c.kind = K_ADD_I64; c.is_one = 1; c.xform = X_NONE;
        int seen = b.add_slot(c);
        outs.push_back({E_MINMAX, src_type, main, seen, s.xform, true, src_type == SB_DECIMAL64 ? src_scale : 0});
        break;
      }
      case SB_AGG_VAR_POP: case SB_AGG_VAR_SAMP: case SB_AGG_STDDEV_POP: case SB_AGG_STDDEV_SAMP: {
        // CentralMomentAgg: pass 1 (these slots) gives each group's count, mean and range, pass 2 (csrc/moments.cu) the deviations
        SB_REQUIRE((sp.flags & ~SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO) == 0, "unknown aggregate flags %d", sp.flags);
        MomentInput mi;
        memset(&mi, 0, sizeof(mi));
        auto col_slot = [](const Column &c, const uint8_t *valid, int kind, int xform) {
          HostSlot s;
          s.nf = 1;
          s.f[0].data = c.d(); s.f[0].valid = valid; s.f[0].type = c.type; s.f[0].mode = F_COL;
          s.kind = kind; s.xform = xform;
          return s;
        };
        if (final_mode) {   // buffers (n, avg, m2): SUM(n), SUM(n * avg), MIN / MAX(avg) over the non-empty partials
          SB_REQUIRE(next_buf_col + 2 < (int)in->cols.size(), "Final aggregate: a variance / stddev buffer is (n, avg, m2) at column %d", next_buf_col);
          const Column &nc = in->cols[next_buf_col], &ac = in->cols[next_buf_col + 1], &mc = in->cols[next_buf_col + 2];
          SB_REQUIRE(nc.type == SB_FLOAT64 && ac.type == SB_FLOAT64 && mc.type == SB_FLOAT64, "variance / stddev buffers (n, avg, m2) must be float64");
          next_buf_col += 3;
          Column n_m, avg_m;
          moments_mask_buffers(nc, ac, mc, n_m, avg_m, st);
          b.temps.push_back(n_m);
          b.temps.push_back(avg_m);
          mi.x = avg_m.d(); mi.xv = avg_m.v(); mi.xtype = SB_FLOAT64;
          mi.n = (const double *)n_m.d(); mi.m2 = (const double *)mc.d();
          mi.slot_cnt = b.add_slot(col_slot(n_m, nullptr, K_ADD_F64, X_NONE));
          HostSlot prod = col_slot(n_m, nullptr, K_ADD_F64, X_NONE);
          prod.nf = 2;
          prod.f[1] = col_slot(avg_m, avg_m.v(), K_ADD_F64, X_NONE).f[0];
          mi.slot_sum = b.add_slot(prod);
          mi.slot_min = b.add_slot(col_slot(avg_m, avg_m.v(), K_MIN_U64, X_DOUBLE));
          mi.slot_max = b.add_slot(col_slot(avg_m, avg_m.v(), K_MAX_U64, X_DOUBLE));
        } else {            // the input as DOUBLE: COUNT, SUM, MIN, MAX of x
          int c;
          Column src;
          const sb_expr &e = sp.input;
          if (expr_is_column(e, &c) || (e.n == 2 && e.nodes[0].op == SB_OP_COL && e.nodes[1].op == SB_OP_CAST_F64 && (c = e.nodes[0].arg, true))) {
            SB_REQUIRE(c >= 0 && c < (int)in->cols.size(), "aggregate input column %d out of range", c);
            src = in->cols[c];   // a numeric column is read as double in the kernels: what Cast(_, DoubleType) does
          } else {
            expr_validate(in, e);
            src = eval_projection(in, e, nullptr, in->nrows, st);
            b.temps.push_back(src);
          }
          if (src.type < SB_INT8 || src.type > SB_FLOAT64) fail(SB_ERR_UNSUPPORTED, "variance / stddev of a column of type %d is not supported", src.type);
          const uint8_t *valid = nulls_of(src);
          mi.x = src.d(); mi.xv = valid; mi.xtype = src.type;
          HostSlot cnt = col_slot(src, valid, K_ADD_I64, X_NONE);
          cnt.is_one = 1;
          mi.slot_cnt = b.add_slot(cnt);
          mi.slot_sum = b.add_slot(col_slot(src, valid, K_ADD_F64, X_NONE));
          mi.slot_min = b.add_slot(col_slot(src, valid, K_MIN_U64, X_DOUBLE));
          mi.slot_max = b.add_slot(col_slot(src, valid, K_MAX_U64, X_DOUBLE));
        }
        MomentOut mo;
        memset(&mo, 0, sizeof(mo));
        mo.input = -1;
        for (size_t j = 0; j < mom_in.size(); j++)   // var(x) and stddev(x) share their passes
          if (mom_in[j].slot_cnt == mi.slot_cnt && mom_in[j].slot_sum == mi.slot_sum && mom_in[j].slot_min == mi.slot_min &&
              mom_in[j].slot_max == mi.slot_max)
            mo.input = (int32_t)j;
        if (mo.input < 0) {
          mo.input = (int32_t)mom_in.size();
          mom_in.push_back(mi);
        }
        mo.func = sp.func;
        mo.flags = sp.flags;
        mom_out.push_back(mo);
        mom_first_out.push_back((int)outs.size());
        for (int k = 0; k < (emit_buffers ? 3 : 1); k++) outs.push_back({OUT_MOMENT, SB_FLOAT64, -1, -1, X_NONE, !emit_buffers});
        break;
      }
      default: fail(SB_ERR_INVALID, "unknown aggregate function %d", sp.func);
    }
  }
  // ---- columns: canonical numbering (mask, filter terms, keys, slot factors) -------------------------------------
  if (m.has_mask) m.mask_col = col_index(mask_ref.data, mask_ref.valid, mask_ref.type);
  for (int i = 0; i < m.nterms; i++) m.term_col[i] = col_index(term_refs[i].data, term_refs[i].valid, term_refs[i].type);
  for (int i = 0; i < m.nkeys; i++) m.key_col[i] = col_index(key_refs[i].data, key_refs[i].valid, key_refs[i].type);
  // ---- slots -> PlanMeta + argument arrays -----------------------------------------------------------------
  m.nslots = (int)b.slots.size();
  for (int i = 0; i < m.nslots; i++) {
    const HostSlot &sl = b.slots[i];
    m.slot_kind[i] = sl.kind; m.slot_nf[i] = sl.nf; m.slot_one[i] = sl.is_one; m.slot_xform[i] = sl.xform;
    m.slot_cls[i] = CLS_GENERIC;
    bool any_valid = false, plain = sl.nf >= 1;
    for (int k = 0; k < sl.nf; k++) {
      m.f_col[i][k] = col_index(sl.f[k].data, sl.f[k].valid, sl.f[k].type);
      a.fac_lit[i][k] = sl.f[k].lit;
      m.f_type[i][k] = sl.f[k].type; m.f_mode[i][k] = sl.f[k].mode; m.f_valid[i][k] = sl.f[k].valid != nullptr;
      any_valid |= sl.f[k].valid != nullptr;
      plain &= sl.f[k].type == SB_FLOAT64 && sl.f[k].valid == nullptr;
    }
    m.slot_anyvalid[i] = any_valid;
    if (sl.is_one && sl.nf == 0 && sl.kind == K_ADD_I64) m.slot_cls[i] = CLS_ONE;
    if (!sl.is_one && sl.kind == K_ADD_F64 && sl.xform == X_NONE && plain) m.slot_cls[i] = CLS_F64_PRODUCT;
  }
  const int ns = m.nslots;

  // ---- launch geometry -------------------------------------------------------------------------------------
  int64_t cap_max = next_pow2(n > 512 ? 2 * n : 1024);
  // no hint: 128K groups before the first retry -- except for inputs small enough that a table for "every row its own group"
  // costs less to clear than a failed attempt costs to run (the join outputs Q3 / Q5 aggregate, a Final over Partial rows)
  int64_t cap = plan->expected_groups > 0 ? next_pow2(4 * plan->expected_groups) : (n <= (1 << 23) ? cap_max : (1 << 18));
  if (cap < 1024) cap = 1024;
  if (cap > cap_max) cap = cap_max;
  auto dict_smem = [&](int d) { return (size_t)(d + 1 + (size_t)(d + 1) * ns * AGG_THREADS) * 8; };
  auto dict_blocks_per_sm = [&](int d) {
    int b = (int)((228 * 1024) / (dict_smem(d) + 1024));
    return b < 1 ? 1 : (b > 8 ? 8 : b);
  };
  // which members of the kernel family this call can reach (only those are specialised at run time)
  const bool light_plan = dict_blocks_per_sm(8) == dict_blocks_per_sm(4), big_dict_ok = dict_blocks_per_sm(32) >= 4;
  int need = light_plan ? (NEED_K1W | (big_dict_ok ? NEED_K2B : 0) | NEED_SMEM) : (NEED_K1 | NEED_K2 | NEED_SMEM);
  if (config().agg_tier == 1 || (config().agg_tier == 0 && plan->expected_groups > 0 && plan->expected_groups <= AGG_DICT)) need = NEED_DIRECT;
  else if (config().agg_tier == 2 || (config().agg_tier == 0 && plan->expected_groups > AGG_DICT)) need = NEED_SMEM;
  KernelChoice kc = choose_kernels(m, a.nwords == 1 ? n : 0, need);   // wide-key kernels are not specialised
  const size_t smem_acc = (size_t)(AGG_DICT + 1 + (size_t)(AGG_DICT + 1) * ns * AGG_THREADS) * 8;   // dictionary + fill counter + accumulators
  SB_REQUIRE(smem_acc <= 200 * 1024, "aggregate needs %zu bytes of shared memory", smem_acc);
  SB_CUDA(cudaFuncSetAttribute(kc.direct, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_acc));
  // persistent grids are sized from the kernel's REAL residency (registers may allow fewer blocks than shared memory does: a
  // grid of 8 blocks per SM over a kernel that fits 6 runs a second, mostly idle wave)
  auto resident_blocks = [&](AggKernel k, size_t smem, int upper) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k, AGG_THREADS, smem) != cudaSuccess || nb < 1) {
      cudaGetLastError();
      nb = 1;
    }
    return nb < upper ? nb : upper;
  };
  int blocks_per_sm = resident_blocks(kc.direct, smem_acc, dict_blocks_per_sm(AGG_DICT));
  int grid = grid_for(n, AGG_THREADS * kc.items_direct, rt().num_sms * blocks_per_sm);
  // the automatic chain's geometry (k1 defines the tiles; k2 walks k1's tiles with fewer, fatter blocks)
  if (kc.k1_wide && light_plan) {   // light plan: the 8-entry dictionary costs no occupancy, so
    kc.k1 = kc.k1_wide;                                                 // it goes first and a 32-entry one (if it keeps >= 4
    kc.k1_dict = 8;                                                     // blocks per SM) catches 9..32 groups before the
    kc.k2 = nullptr;                                                    // shared-memory tier and its atomics
    if (kc.k2_big && big_dict_ok) {
      kc.k2 = kc.k2_big;
      kc.k2_dict = 32;
    }
  }
  const size_t smem_k1 = dict_smem(kc.k1_dict), smem_k2 = dict_smem(kc.k2_dict);
  SB_CUDA(cudaFuncSetAttribute(kc.k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k1));
  if (kc.k2) SB_CUDA(cudaFuncSetAttribute(kc.k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k2));
  const int grid_k1 = grid_for(n, AGG_THREADS * kc.k1_items, rt().num_sms * resident_blocks(kc.k1, smem_k1, dict_blocks_per_sm(kc.k1_dict)));
  const int grid_k2 = kc.k2 ? std::min(grid_k1, rt().num_sms * resident_blocks(kc.k2, smem_k2, dict_blocks_per_sm(kc.k2_dict))) : 0;
  // ---- tiers: "dict" (lane-private dictionary + HBM table), "smem" (shared-memory table + HBM table), or "auto": the
  // dictionary kernel starts, yields as soon as the input turns out not to be a few-groups shape, and the shared-memory kernel
  // launched behind it finishes the job (AggArgs::gate) -- no sample pass, no host round trip.
  int tier = config().agg_tier;   // 0 auto, 1 dict only, 2 smem only (tests force a tier through sb_config_set)
  int32_t scap = 8192;
  while (scap > 512 && (size_t)(scap + 2) * (1 + ns) * 8 + 64 > 200 * 1024) scap >>= 1;
  // tiny inputs (the Final stage of a few-group aggregate: a handful of rows) are pure latency: one block, rows straight into
  // the HBM table -- no dictionary to initialise and merge, no chain of launches
  const bool tiny = tier == 0 && n <= AGG_THREADS * ITEMS_SMEM * AGGS_SUB;
  if (tiny) {
    tier = 2;
    scap = 512;
  }
  a.start_bypassed = tiny ? 1 : 0;
  if (tier == 0 && plan->expected_groups > 0)   // the caller knows: few -> dictionary, else the shared-memory kernel (which bypasses its table when the hit rate is poor)
    tier = plan->expected_groups <= AGG_DICT ? 1 : 2;
  const size_t smem_tab = (size_t)(scap + 2) * (1 + ns) * 8 + 64;
  a.combine = 0;   // any compare-and-swap accumulator kind?
  for (int i = 0; i < ns; i++) a.combine |= m.slot_kind[i] != K_ADD_I64;
  const int grid_smem = grid_for(n, AGG_THREADS * ITEMS_SMEM * AGGS_SUB, rt().num_sms);
  if (tier != 1) SB_CUDA(cudaFuncSetAttribute(kc.smem, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  a.scap = scap;

  Scratch flags(32, st), progress((int64_t)grid_k1 * (AGG_THREADS / 32) * 4 + 16, st), progress2((int64_t)grid_k1 * (AGG_THREADS / 32) * 4 + 16, st);
  std::unique_ptr<Scratch> slot_ids_buf;
  int64_t ngroups = 0;
  void *tkeys = nullptr, *tacc = nullptr;
  struct TableFree {
    void *&k, *&v;
    cudaStream_t st;
    ~TableFree() {
      if (k) cudaFreeAsync(k, st);
      if (v) cudaFreeAsync(v, st);
    }
  } table_free_guard{tkeys, tacc, st};

  // ---- update, retrying with a larger table when probing gives up ------------------------------------------------
  for (;;) {
    int64_t slots = cap + 2;
    SB_CUDA(cudaMallocAsync(&tkeys, (size_t)slots * 8 * a.nwords, st));
    SB_CUDA(cudaMallocAsync(&tacc, (size_t)slots * 8 * (ns ? ns : 1), st));
    SB_CUDA(cudaMemsetAsync(tkeys, 0xff, (size_t)slots * 8 * a.nwords, st));
    SB_CUDA(cudaMemsetAsync(tacc, 0, (size_t)slots * 8 * (ns ? ns : 1), st));
    for (int s = 0; s < ns; s++)
      if (m.slot_kind[s] == K_MIN_U64) SB_CUDA(cudaMemsetAsync((uint64_t *)tacc + (int64_t)s * slots, 0xff, (size_t)slots * 8, st));
    SB_CUDA(cudaMemsetAsync(flags.ptr, 0, 32, st));
    a.tkeys = (uint64_t *)tkeys;
    a.tacc = (uint64_t *)tacc;
    a.flags = flags.as<int32_t>();
    a.cap = cap;
    if (n > 0) {
      KernelTimer kt(final_mode ? "agg_update_final" : "agg_update", st);
      a.gate = 0;
      if (a.nwords == 1 && tier == 1) launch_agg(kc.direct, grid, AGG_THREADS, smem_acc, st, a);
      else if (a.nwords == 1 && tier == 2) launch_agg(kc.smem, grid_smem, AGGS_THREADS, smem_tab, st, a);
      else if (a.nwords == 1) {
        a.gate = 1;
        a.progress = progress.as<int32_t>();
        a.progress2 = kc.k2 ? progress2.as<int32_t>() : progress.as<int32_t>();
        a.last_flag = kc.k2 ? 7 : 6;
        a.dict_grid = grid_k1;
        a.dict_items = kc.k1_items;
        launch_agg(kc.k1, grid_k1, AGG_THREADS, smem_k1, st, a);
        SB_LAUNCH_CHECK();
        if (kc.k2) {
          launch_agg(kc.k2, grid_k2, AGG_THREADS, smem_k2, st, a);
          SB_LAUNCH_CHECK();
        }
        a.gate = 2;
        launch_agg(kc.smem, grid_smem, AGGS_THREADS, smem_tab, st, a);
      }
      else if (a.nwords == 2) agg_update_wide_kernel<2, 4><<<grid, AGG_THREADS, 0, st>>>(a);
      else if (a.nwords == 3) agg_update_wide_kernel<3, 4><<<grid, AGG_THREADS, 0, st>>>(a);
      else agg_update_wide_kernel<4, 4><<<grid, AGG_THREADS, 0, st>>>(a);
      SB_LAUNCH_CHECK();
    }
    // occupied slots -> dense list; the abort flag and the group count come back with ONE host round trip
    {
      const int64_t slots_now = cap + 2;
      slot_ids_buf.reset(new Scratch(slots_now * 8, st));
      Scratch occ(slots_now + 16, st), f32(compact_tiles(slots_now) * 4 + 16, st), pos(compact_tiles(slots_now) * 8 + 16, st);
      occupied_kernel<<<(unsigned)((slots_now + 255) / 256), 256, 0, st>>>((uint64_t *)tkeys, cap, flags.as<int32_t>(), occ.as<uint8_t>());
      SB_LAUNCH_CHECK();
      compact_mask_async(occ.as<uint8_t>(), slots_now, slot_ids_buf->as<int64_t>(), f32.as<int32_t>(), pos.as<int64_t>(),
                         (int64_t *)((char *)flags.ptr + 16), st);
      int64_t host_buf[3];
      SB_CUDA(cudaMemcpyAsync(host_buf, flags.ptr, 24, cudaMemcpyDeviceToHost, st));
      SB_CUDA(cudaStreamSynchronize(st));
      int32_t hflags[4];
      memcpy(hflags, host_buf, 16);
      ngroups = host_buf[2];
      if (!hflags[0]) break;
    }
    if (cap >= cap_max) fail(SB_ERR_CUDA, "hash aggregate table overflow at maximum capacity %lld", (long long)cap);
    cudaFreeAsync(tkeys, st); tkeys = nullptr;
    cudaFreeAsync(tacc, st); tacc = nullptr;
    cap = cap * 16 > cap_max ? cap_max : cap * 16;
  }
  g_last_plan_name = kc.name;
  if (config().agg_verbose) fprintf(stderr, "[sb_hash_aggregate] n=%lld plan=%s path=%s tier=%s cap=%lld slots=%d scap=%d\n", (long long)n, kc.name.c_str(),
                                        a.nwords > 1 ? "wide" : "direct", tier == 0 ? "auto" : (tier == 1 ? "dict" : "smem"),
                                        (long long)cap, ns, scap);
  Scratch &slot_ids = *slot_ids_buf;
  if (plan->nkeys == 0 && ngroups == 0) {
    // no grouping keys: exactly one output row even for empty input (AggregateCodegenSupport.scala:131);
    // slot 0 of the untouched table holds the identities
    SB_CUDA(cudaMemsetAsync(slot_ids.ptr, 0, 8, st));
    ngroups = 1;
  }

  // ---- emit -------------------------------------------------------------------------------------
  sb_table *t = table_new(ngroups);
  try {
    static thread_local EmitArgs emit_storage;
    EmitArgs &e = emit_storage;
    memset(&e, 0, sizeof(e));
    e.nkeys = plan->nkeys;
    e.single64 = m.single64;
    e.nwords = a.nwords;
    e.tkeys = (const uint64_t *)tkeys;
    e.tacc = (const uint64_t *)tacc;
    e.slot_ids = slot_ids.as<int64_t>();
    e.cap = cap;
    e.ngroups = ngroups;
    for (int k = 0; k < plan->nkeys; k++) {
      const Column &src = in->cols[plan->key_cols[k]];
      Column c = column_alloc(src.type, src.scale, ngroups, m.key_valid[k] != 0, st);
      t->cols.push_back(c);
      e.key[k].out = c.data->ptr;
      e.key[k].out_valid = c.validity ? (uint32_t *)c.validity->ptr : nullptr;
      e.key[k].type = src.type;
      e.key[k].bits = m.key_bits[k];
      e.key[k].shift = m.key_shift[k];
      e.key[k].null_shift = m.key_nshift[k];
      e.key[k].word = a.key_extra[k].word;
      e.key[k].null_word = a.key_extra[k].null_word;
      e.key[k].hi_word = a.key_extra[k].hi_word;
      e.key[k].hi_shift = a.key_extra[k].hi_shift;
    }
    e.ncols = 0;
    for (size_t i = 0; i < outs.size(); i++) {
      Column c = column_alloc(outs[i].out_type, outs[i].scale, ngroups, outs[i].nullable, st);
      t->cols.push_back(c);
      if (outs[i].op == OUT_MOMENT) continue;
      SB_REQUIRE(e.ncols < 2 * AGG_MAX_SLOTS, "too many aggregate output columns");
      EmitCol &ec = e.col[e.ncols++];
      ec.out = c.data->ptr;
      ec.out_valid = c.validity ? (uint32_t *)c.validity->ptr : nullptr;
      ec.op = outs[i].op;
      ec.out_type = outs[i].out_type;
      ec.slot = outs[i].slot;
      ec.slot2 = outs[i].slot2;
      ec.xform = outs[i].xform;
    }
    if (ngroups > 0) {
      agg_emit_kernel<<<(unsigned)((ngroups + 255) / 256), 256, 0, st>>>(e);
      SB_LAUNCH_CHECK();
    }
    for (size_t j = 0; j < mom_out.size(); j++) {
      const int first = plan->nkeys + mom_first_out[j];
      for (int k = 0; k < (emit_buffers ? 3 : 1); k++) mom_out[j].out[k] = t->cols[first + k].data->ptr;
      mom_out[j].out_valid = emit_buffers ? nullptr : (uint32_t *)t->cols[first].validity->ptr;
    }
    moments_run(a, mom_in, mom_out, final_mode, emit_buffers, slot_ids.as<int64_t>(), ngroups, st);
    // no host synchronisation: the table buffers stay valid until after the emit kernel in stream order
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
}

}  // namespace sb

using namespace sb;

// Compile check of the run-time specialisation for a PlanMeta given as raw int32 words (no device needed): used by the
// CPU-side build check so that a header change that breaks NVRTC compilation is caught without a GPU.
extern "C" int sb_agg_rtc_compile_check(const int32_t *plan_meta_words, int32_t nwords, char *log, int32_t log_len) {
  SB_API_BEGIN
  SB_REQUIRE(plan_meta_words && nwords == (int32_t)(sizeof(PlanMeta) / 4), "expected %d PlanMeta words, got %d", (int)(sizeof(PlanMeta) / 4), nwords);
  PlanMeta m;
  memcpy(&m, plan_meta_words, sizeof(m));
  const void *k[6];
  std::string lg;
  const bool ok = specialise_kernels(m, chain_items(m), NEED_ALL, false, k, &lg, nullptr);
  if (log && log_len > 0) snprintf(log, (size_t)log_len, "%s", lg.c_str());
  if (!ok) fail(SB_ERR_UNSUPPORTED, "run-time compilation failed: %s", lg.c_str());
  SB_API_END
}
extern "C" int32_t sb_agg_plan_meta_words(void) { return (int32_t)(sizeof(PlanMeta) / 4); }

// String grouping keys (HashAggregateExec groups UTF8String keys by their bytes): the key column is replaced by its
// order-preserving dictionary codes (csrc/strings.cu), the fixed-width kernels group the codes, and the key columns of the result
// are decoded back.  Every mode works the same way -- a Final / PartialMerge input carries decoded strings again.
static void hash_aggregate_strings(const sb_table *in, const sb_agg_plan *plan, cudaStream_t st, sb_table **out);
// decimal SUM / AVG first (limb sums around the aggregate, csrc/decimal.cu), then string keys (dictionary codes), then the kernels
static void hash_aggregate_impl(const sb_table *in, const sb_agg_plan *plan, cudaStream_t st, sb_table **out) {
  SB_REQUIRE(in && plan && out, "null argument");
  if (plan_has_decimal_sums(in, plan)) {
    hash_aggregate_decimals(in, plan, st, hash_aggregate_strings, out);
    return;
  }
  hash_aggregate_strings(in, plan, st, out);
}
static void hash_aggregate_strings(const sb_table *in, const sb_agg_plan *plan, cudaStream_t st, sb_table **out) {
  SB_REQUIRE(in && plan && out, "null argument");
  std::vector<int> scols;
  for (int k = 0; k < plan->nkeys; k++) {
    const int ci = plan->key_cols[k];
    if (ci >= 0 && ci < (int)in->cols.size() && in->cols[ci].type == SB_STRING) scols.push_back(ci);
  }
  if (scols.empty()) {
    hash_aggregate_fixed(in, plan, st, out);
    return;
  }
  EncodedView ev;
  encode_string_columns(in, scols, nullptr, st, ev);
  sb_table *res = nullptr;
  hash_aggregate_fixed(ev.view, plan, st, &res);
  try {
    for (int k = 0; k < plan->nkeys; k++) {
      const Column *dict = ev.dictionary_of(plan->key_cols[k]);
      if (!dict) continue;
      Column decoded = dictionary_decode(res->cols[k], *dict, st);
      column_release(res->cols[k]);
      res->cols[k] = decoded;
    }
  } catch (...) {
    table_free(res);
    throw;
  }
  *out = res;
}

// which kernels the calling thread's last sb_hash_aggregate ran: "generic" or "rtc:<plan hash>[(disk)]"
extern "C" const char *sb_hash_aggregate_last_plan(void) { return g_last_plan_name.c_str(); }

extern "C" int sb_hash_aggregate(const sb_table *in, const sb_agg_plan *plan, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  hash_aggregate_impl(in, plan, stream_of(s), out);
  SB_API_END
}

// ---- aggregation state across an iterator of batches ----------------------------------------------------------------
// TungstenAggregationIterator.processInputs (TungstenAggregationIterator.scala:206-281) folds every input row of the
// partition into one map.  Here each batch is aggregated on its own (one pass, the kernels above) into a Partial table
// (keys ++ buffers) that is parked in the state; parked tables are merged (PartialMerge: buffers -> buffers) whenever
// they add up to more than kCompactRows rows, and once more in finish().  Nothing is concatenated at input size: a batch
// can be released as soon as update() returns, and HBM holds one batch plus the groups seen so far.
struct sb_agg_state {
  sb_agg_plan plan;                       // deep copy (the arrays below back its pointers)
  std::vector<int32_t> key_cols;
  std::vector<sb_agg_spec> aggs;
  std::vector<std::vector<sb_expr_node>> nodes;
  std::vector<std::vector<uint8_t>> bytes;   // string literal pools of the inputs
  sb_expr filter;
  std::vector<sb_expr_node> filter_nodes;
  std::vector<uint8_t> filter_bytes;
  std::vector<int32_t> merged_keys;       // 0..nkeys-1: where the keys sit in a Partial table
  std::vector<sb_table *> parked;
  int64_t parked_rows = 0;
  std::mutex mu;
};
static constexpr int64_t kCompactRows = 1 << 22;
static constexpr size_t kCompactTables = 64;

static sb_table *agg_state_merge(sb_agg_state *st, int mode, cudaStream_t cs) {   // all parked tables -> one table of `mode`
  sb_table *cat = nullptr;
  if (st->parked.size() == 1) {
    cat = st->parked[0];
    cat->refs.fetch_add(1);
  } else {
    sb_stream tmp;
    tmp.stream = cs;
    int rc = sb_table_concat(st->parked.data(), (int32_t)st->parked.size(), &tmp, &cat);
    if (rc != SB_OK) fail(rc, "%s", sb_last_error());
  }
  sb_agg_plan p = st->plan;
  p.mode = mode;
  p.key_cols = st->merged_keys.data();
  p.filter = nullptr;
  sb_table *out = nullptr;
  try {
    hash_aggregate_impl(cat, &p, cs, &out);
  } catch (...) {
    sb_table_release(cat);
    throw;
  }
  sb_table_release(cat);
  return out;
}

extern "C" int sb_hash_agg_create(const sb_agg_plan *plan, sb_agg_state **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(plan && out, "null argument");
  SB_REQUIRE(plan->mode >= SB_AGG_MODE_PARTIAL && plan->mode <= SB_AGG_MODE_PARTIAL_MERGE, "bad aggregate mode %d", plan->mode);
  SB_REQUIRE(plan->nkeys >= 0 && plan->naggs >= 0 && plan->nkeys <= AGG_MAX_KEYS, "bad plan");
  std::unique_ptr<sb_agg_state> st(new sb_agg_state());
  st->plan = *plan;
  st->key_cols.assign(plan->key_cols, plan->key_cols + plan->nkeys);
  st->aggs.assign(plan->aggs, plan->aggs + plan->naggs);
  st->nodes.resize(plan->naggs);
  st->bytes.resize(plan->naggs);
  auto copy_pool = [](const sb_expr &e, std::vector<uint8_t> &to, sb_expr &copy) {
    if (e.bytes && e.nbytes > 0) to.assign(e.bytes, e.bytes + e.nbytes);
    copy.bytes = to.empty() ? nullptr : to.data();
  };
  for (int i = 0; i < plan->naggs; i++) {
    const sb_expr &e = plan->aggs[i].input;
    if (e.nodes && e.n > 0) {
      st->nodes[i].assign(e.nodes, e.nodes + e.n);
      st->aggs[i].input.nodes = st->nodes[i].data();
      copy_pool(e, st->bytes[i], st->aggs[i].input);
    } else {
      st->aggs[i].input.nodes = nullptr;
      st->aggs[i].input.n = 0;
    }
  }
  st->plan.key_cols = st->key_cols.data();
  st->plan.aggs = st->aggs.data();
  st->plan.filter = nullptr;
  if (plan->filter) {
    st->filter_nodes.assign(plan->filter->nodes, plan->filter->nodes + plan->filter->n);
    st->filter = *plan->filter;
    st->filter.nodes = st->filter_nodes.data();
    copy_pool(*plan->filter, st->filter_bytes, st->filter);
    st->plan.filter = &st->filter;
  }
  for (int i = 0; i < plan->nkeys; i++) st->merged_keys.push_back(i);
  *out = st.release();
  SB_API_END
}

static void agg_state_park(sb_agg_state *st, sb_table *t, cudaStream_t cs) {
  st->parked.push_back(t);
  st->parked_rows += t->nrows;
  if (st->parked.size() > 1 && (st->parked_rows > kCompactRows || st->parked.size() >= kCompactTables)) {
    sb_table *m = agg_state_merge(st, SB_AGG_MODE_PARTIAL_MERGE, cs);
    for (auto *p : st->parked) sb_table_release(p);
    st->parked.clear();
    st->parked.push_back(m);
    st->parked_rows = m->nrows;
  }
}

extern "C" int sb_hash_agg_update(sb_agg_state *st, const sb_table *batch, sb_stream *s) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(st && batch, "null argument");
  std::lock_guard<std::mutex> lk(st->mu);
  cudaStream_t cs = stream_of(s);
  sb_table *part = nullptr;
  if (st->plan.mode == SB_AGG_MODE_FINAL || st->plan.mode == SB_AGG_MODE_PARTIAL_MERGE) {
    // the input already is keys ++ buffers: bring the keys to the front so that parked tables share one layout
    sb_agg_plan p = st->plan;
    p.mode = SB_AGG_MODE_PARTIAL_MERGE;
    hash_aggregate_impl(batch, &p, cs, &part);
  } else {
    sb_agg_plan p = st->plan;
    p.mode = SB_AGG_MODE_PARTIAL;
    hash_aggregate_impl(batch, &p, cs, &part);
  }
  agg_state_park(st, part, cs);
  SB_API_END
}

extern "C" int sb_hash_agg_merge(sb_agg_state *st, const sb_table *partial, sb_stream *s) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(st && partial, "null argument");
  std::lock_guard<std::mutex> lk(st->mu);
  sb_table *t = const_cast<sb_table *>(partial);   // keys ++ buffers in Partial layout (another state's finish, an exchange)
  t->refs.fetch_add(1);
  agg_state_park(st, t, stream_of(s));
  SB_API_END
}

extern "C" int sb_hash_agg_finish(sb_agg_state *st, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(st && out, "null argument");
  std::lock_guard<std::mutex> lk(st->mu);
  SB_REQUIRE(!st->parked.empty(), "sb_hash_agg_finish before any batch (pass an empty batch for an empty partition)");
  const bool results = st->plan.mode == SB_AGG_MODE_FINAL || st->plan.mode == SB_AGG_MODE_COMPLETE;
  *out = agg_state_merge(st, results ? SB_AGG_MODE_FINAL : SB_AGG_MODE_PARTIAL_MERGE, stream_of(s));
  SB_API_END
}

extern "C" int sb_hash_agg_destroy(sb_agg_state *st) {
  SB_API_BEGIN
  if (st) {
    for (auto *p : st->parked) sb_table_release(p);
    delete st;
  }
  SB_API_END
}
