// expr.cu -- generic (unfused) evaluation of FilterExec / ProjectExec expression programs.
//
// Reference semantics restated (no code shared): sql/catalyst/.../expressions/arithmetic.scala
// (Add/Subtract/Multiply wrap in non-ANSI mode; Divide is double division, NULL on a zero divisor),
// predicates.scala (And/Or are Kleene three-valued; comparisons are NULL when an operand is NULL),
// SQLOrderingUtil.compareDoubles (NaN == NaN, NaN is the largest double, -0.0 == 0.0),
// FilterExec keeps a row only when the predicate is TRUE (SQLX/basicPhysicalOperators.scala:245).
//
// This is the general path: one pass per expression, results materialised as columns.  Hot fused
// shapes (TPC-H stages) bypass it -- see aggregate.cu.
#include <vector>
#include "expr.cuh"
#include "simple_pred.cuh"
#include "strpred.cuh"
#include "primitives.cuh"
#include "rtc.cuh"

namespace sb {

constexpr int EXPR_MAX_COLS = 12;

struct DevNode {
  int32_t op, vtype, arg, arg2;
  int64_t lit;   // string tests: the descriptor's word index in `blob`
};
struct DevProg {
  int32_t n;
  int32_t ncols;
  DevNode nodes[EXPR_MAX_NODES];
  const void *col_data[EXPR_MAX_COLS];
  const uint8_t *col_valid[EXPR_MAX_COLS];
  const int32_t *col_offsets[EXPR_MAX_COLS];   // string columns
  int32_t col_type[EXPR_MAX_COLS];
  const uint32_t *blob;                        // the program's string literals (strpred.cuh), or null
};

static int vtype_of_column(int32_t t) {
  switch (t) {
    case SB_BOOL: return SB_VT_BOOL;
    case SB_INT8: case SB_INT16: case SB_INT32: case SB_DATE32: return SB_VT_I32;
    case SB_INT64: case SB_TIMESTAMP: case SB_DECIMAL64: return SB_VT_I64;
    case SB_FLOAT32: case SB_FLOAT64: return SB_VT_F64;
  }
  return 0;
}

bool expr_is_column(const sb_expr &e, int *col) {
  if (e.n == 1 && e.nodes[0].op == SB_OP_COL) {
    if (col) *col = e.nodes[0].arg;
    return true;
  }
  return false;
}

void expr_validate(const sb_table *in, const sb_expr &e) {
  SB_REQUIRE(e.nodes && e.n >= 1 && e.n <= EXPR_MAX_NODES, "expression must have 1..%d nodes (got %d)", EXPR_MAX_NODES, e.n);
  int depth = 0;
  // Decimal columns carry unscaled integers: arithmetic and comparisons on them would need the rescaling / precision rules of
  // DecimalPrecision (sql/catalyst/.../analysis/DecimalPrecision.scala) and are rejected rather than evaluated on the unscaled
  // values (ADVICE round 1: they used to be silently wrong).  Bare references and IS [NOT] NULL are fine.
  bool has_decimal = false, only_null_tests = true;
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    if (nd.op == SB_OP_COL && nd.arg >= 0 && nd.arg < (int)in->cols.size() && (in->cols[nd.arg].type == SB_DECIMAL64 || in->cols[nd.arg].type == SB_DECIMAL128)) has_decimal = true;
    if (nd.op != SB_OP_COL && nd.op != SB_OP_ISNULL && nd.op != SB_OP_ISNOTNULL && nd.op != SB_OP_AND && nd.op != SB_OP_OR && nd.op != SB_OP_NOT)
      only_null_tests = false;
  }
  if (has_decimal && e.n > 1 && !only_null_tests)
    fail(SB_ERR_UNSUPPORTED, "arithmetic / comparison on DECIMAL columns is not implemented on the GPU path (unscaled values would ignore the scale)");
  // Type check: the kernels trust the vtypes (a CAST reads its source class from `arg`, a comparison compares as `arg`, arithmetic
  // works at the node's vtype), so a program whose operands disagree with them would be evaluated on reinterpreted bits.  vt[] is
  // the class of each stack slot; a NULL literal (null_lit[]) is accepted in any class.
  int32_t vt[EXPR_STACK + 1];
  bool null_lit[EXPR_STACK + 1];
  int cols_seen[EXPR_MAX_COLS], ncols = 0;
  auto operand_ok = [&](int slot, int32_t want) { return null_lit[slot] || vt[slot] == want; };
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    int32_t res = nd.vtype;
    switch (nd.op) {
      case SB_OP_COL: {
        SB_REQUIRE(nd.arg >= 0 && nd.arg < (int)in->cols.size(), "expression references column %d of %zu", nd.arg, in->cols.size());
        int32_t t = in->cols[nd.arg].type;
        if (t == SB_STRING) {
          if (e.n != 1) fail(SB_ERR_UNSUPPORTED, "string columns are only supported as bare references in expressions");
        } else {
          SB_REQUIRE(nd.vtype == vtype_of_column(t), "COL node %d: vtype %d does not match column type %d", i, nd.vtype, t);
        }
        bool seen = false;
        for (int c = 0; c < ncols; c++) seen |= cols_seen[c] == nd.arg;
        if (!seen) {
          SB_REQUIRE(ncols < EXPR_MAX_COLS, "expression references more than %d distinct columns", EXPR_MAX_COLS);
          cols_seen[ncols++] = nd.arg;
        }
        break;
      }
      case SB_OP_LIT_I64:
        SB_REQUIRE(nd.vtype >= SB_VT_BOOL && nd.vtype <= SB_VT_I64, "LIT_I64 node %d: vtype %d is not BOOL, I32 or I64", i, nd.vtype);
        break;
      case SB_OP_LIT_F64: SB_REQUIRE(nd.vtype == SB_VT_F64, "LIT_F64 node %d: vtype %d is not F64", i, nd.vtype); break;
      case SB_OP_LIT_NULL:
        SB_REQUIRE(nd.vtype >= SB_VT_BOOL && nd.vtype <= SB_VT_F64, "LIT_NULL node %d: unknown vtype %d", i, nd.vtype);
        break;
      case SB_OP_ADD: case SB_OP_SUB: case SB_OP_MUL: case SB_OP_DIV:
      case SB_OP_EQ: case SB_OP_NE: case SB_OP_LT: case SB_OP_LE: case SB_OP_GT: case SB_OP_GE:
      case SB_OP_AND: case SB_OP_OR: {
        SB_REQUIRE(depth >= 2, "expression stack underflow at node %d", i);
        int32_t want;
        if (nd.op == SB_OP_DIV) {
          want = SB_VT_F64;
          SB_REQUIRE(nd.vtype == SB_VT_F64, "DIV node %d: vtype %d is not F64", i, nd.vtype);
        } else if (nd.op >= SB_OP_ADD && nd.op <= SB_OP_MUL) {
          want = nd.vtype;
          SB_REQUIRE(nd.vtype >= SB_VT_I32 && nd.vtype <= SB_VT_F64, "arithmetic node %d: vtype %d is not numeric", i, nd.vtype);
        } else if (nd.op >= SB_OP_EQ && nd.op <= SB_OP_GE) {
          want = nd.arg;
          SB_REQUIRE(nd.vtype == SB_VT_BOOL, "comparison node %d: vtype %d is not BOOL", i, nd.vtype);
        } else {
          want = SB_VT_BOOL;
          SB_REQUIRE(nd.vtype == SB_VT_BOOL, "AND / OR node %d: vtype %d is not BOOL", i, nd.vtype);
        }
        SB_REQUIRE(operand_ok(depth - 2, want) && operand_ok(depth - 1, want), "node %d (op %d): operands of vtype %d and %d, expected %d", i,
                   nd.op, vt[depth - 2], vt[depth - 1], want);
        depth -= 2;
        break;
      }
      case SB_OP_NEG: case SB_OP_NOT: case SB_OP_ISNULL: case SB_OP_ISNOTNULL:
      case SB_OP_CAST_F64: case SB_OP_CAST_I64: case SB_OP_CAST_I32: {
        SB_REQUIRE(depth >= 1, "expression stack underflow at node %d", i);
        const int32_t src = vt[depth - 1];
        if (nd.op == SB_OP_NEG) {
          SB_REQUIRE(nd.vtype >= SB_VT_I32 && nd.vtype <= SB_VT_F64 && operand_ok(depth - 1, nd.vtype), "NEG node %d: vtype %d over an operand of vtype %d", i,
                     nd.vtype, src);
        } else if (nd.op == SB_OP_NOT) {
          SB_REQUIRE(nd.vtype == SB_VT_BOOL && operand_ok(depth - 1, SB_VT_BOOL), "NOT node %d: vtype %d over an operand of vtype %d", i, nd.vtype, src);
        } else if (nd.op == SB_OP_ISNULL || nd.op == SB_OP_ISNOTNULL) {
          SB_REQUIRE(nd.vtype == SB_VT_BOOL, "IS [NOT] NULL node %d: vtype %d is not BOOL", i, nd.vtype);
        } else {
          res = nd.op == SB_OP_CAST_F64 ? SB_VT_F64 : nd.op == SB_OP_CAST_I64 ? SB_VT_I64 : SB_VT_I32;
          SB_REQUIRE(nd.vtype == res, "CAST node %d: vtype %d, expected %d", i, nd.vtype, res);
          SB_REQUIRE(nd.arg >= SB_VT_BOOL && nd.arg <= SB_VT_F64 && operand_ok(depth - 1, nd.arg),
                     "CAST node %d: arg (source class) %d but the operand has vtype %d", i, nd.arg, src);
        }
        depth--;
        break;
      }
      default: {
        if (!strpred_is_leaf(nd.op)) fail(SB_ERR_INVALID, "unknown expression op %d at node %d", nd.op, i);
        res = strpred_validate(in, e, i);
        bool seen = false;
        for (int c = 0; c < ncols; c++) seen |= cols_seen[c] == nd.arg;
        if (!seen) {
          SB_REQUIRE(ncols < EXPR_MAX_COLS, "expression references more than %d distinct columns", EXPR_MAX_COLS);
          cols_seen[ncols++] = nd.arg;
        }
        break;
      }
    }
    SB_REQUIRE(depth < EXPR_STACK, "expression needs more than %d stack slots", EXPR_STACK);
    vt[depth] = res;
    null_lit[depth] = nd.op == SB_OP_LIT_NULL;
    depth++;
  }
  SB_REQUIRE(depth == 1, "expression leaves %d values on the stack", depth);
}

bool expr_nullable(const sb_table *in, const sb_expr &e) {
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    if ((nd.op == SB_OP_COL || strpred_is_leaf(nd.op)) && in->cols[nd.arg].validity) return true;
    if (nd.op == SB_OP_STR_IN && nd.arg2) return true;
    if (nd.op == SB_OP_DIV || nd.op == SB_OP_LIT_NULL) return true;
  }
  return false;
}

// `e` has passed expr_validate; `tests` / `blob` are its string literals (strpred_compile) and their device copy
static DevProg build_prog(const sb_table *in, const sb_expr &e, const StrTests &tests, const uint32_t *blob) {
  DevProg p;
  p.n = e.n;
  p.ncols = 0;
  p.blob = blob;
  int remap[256];
  for (int i = 0; i < 256; i++) remap[i] = -1;
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    p.nodes[i].op = nd.op;
    p.nodes[i].vtype = nd.vtype;
    p.nodes[i].arg = nd.arg;
    p.nodes[i].arg2 = nd.arg2;
    p.nodes[i].lit = strpred_is_leaf(nd.op) ? (int64_t)tests.ref[i] : nd.lit.i;
    if (nd.op == SB_OP_COL || strpred_is_leaf(nd.op)) {
      SB_REQUIRE(nd.arg < 256, "expression column index too large");
      if (remap[nd.arg] < 0) {
        SB_REQUIRE(p.ncols < EXPR_MAX_COLS, "expression references more than %d distinct columns", EXPR_MAX_COLS);
        const Column &c = in->cols[nd.arg];
        p.col_data[p.ncols] = c.d();
        p.col_valid[p.ncols] = c.v();
        p.col_offsets[p.ncols] = c.o();
        p.col_type[p.ncols] = c.type;
        remap[nd.arg] = p.ncols++;
      }
      p.nodes[i].arg = remap[nd.arg];
    }
  }
  return p;
}

// SQLOrderingUtil.compareDoubles
__device__ __forceinline__ int cmp_f64(double x, double y) {
  if (x == y) return 0;
  bool xn = x != x, yn = y != y;
  if (xn || yn) return (int)xn - (int)yn;
  return x < y ? -1 : 1;
}

// the string tests out of line: inlined, they push eval_row's projection kernel into spilling
__device__ __noinline__ int64_t eval_string_test(int32_t op, uint32_t ref, const uint32_t *blob, const uint8_t *s, int32_t n) {
  return strpred_eval(op, ref, blob, s, n);
}

// evaluates the program for one row; returns raw 64-bit value and null flag
__device__ __forceinline__ void eval_row(const DevProg &p, int64_t row, int64_t &out, bool &out_null) {
  int64_t st[EXPR_STACK];
  bool nl[EXPR_STACK];
  int sp = 0;
#pragma unroll 1
  for (int k = 0; k < p.n; k++) {
    const DevNode nd = p.nodes[k];
    switch (nd.op) {
      case SB_OP_COL: {
        int c = nd.arg;
        bool v = bit_valid(p.col_valid[c], row);
        int64_t x = 0;
        if (v) {
          int t = p.col_type[c];
          if (t == SB_FLOAT32) x = __double_as_longlong((double)((const float *)p.col_data[c])[row]);
          else x = load_i64(p.col_data[c], t, row);
        }
        st[sp] = x; nl[sp] = !v; sp++;
        break;
      }
      case SB_OP_LIT_I64: case SB_OP_LIT_F64: st[sp] = nd.lit; nl[sp] = false; sp++; break;
      case SB_OP_LIT_NULL: st[sp] = 0; nl[sp] = true; sp++; break;
      case SB_OP_ADD: case SB_OP_SUB: case SB_OP_MUL: {
        int64_t b = st[--sp], a = st[sp - 1];
        bool n2 = nl[sp] | nl[sp - 1];
        int64_t r;
        if (nd.vtype == SB_VT_F64) {
          double x = __longlong_as_double(a), y = __longlong_as_double(b);
          double z = nd.op == SB_OP_ADD ? __dadd_rn(x, y) : (nd.op == SB_OP_SUB ? __dsub_rn(x, y) : __dmul_rn(x, y));
          r = __double_as_longlong(z);
        } else {
          uint64_t x = (uint64_t)a, y = (uint64_t)b;
          uint64_t z = nd.op == SB_OP_ADD ? x + y : (nd.op == SB_OP_SUB ? x - y : x * y);
          r = nd.vtype == SB_VT_I32 ? (int64_t)(int32_t)(uint32_t)z : (int64_t)z;   // wrap at the operand width
        }
        st[sp - 1] = r; nl[sp - 1] = n2;
        break;
      }
      case SB_OP_DIV: {
        double y = __longlong_as_double(st[--sp]), x = __longlong_as_double(st[sp - 1]);
        bool n2 = nl[sp] | nl[sp - 1] | (y == 0.0);
        st[sp - 1] = n2 ? 0 : __double_as_longlong(__ddiv_rn(x, y));
        nl[sp - 1] = n2;
        break;
      }
      case SB_OP_NEG: {
        if (nd.vtype == SB_VT_F64) st[sp - 1] = __double_as_longlong(-__longlong_as_double(st[sp - 1]));
        else if (nd.vtype == SB_VT_I32) st[sp - 1] = (int64_t)(int32_t)(0u - (uint32_t)st[sp - 1]);
        else st[sp - 1] = (int64_t)(0ull - (uint64_t)st[sp - 1]);
        break;
      }
      case SB_OP_EQ: case SB_OP_NE: case SB_OP_LT: case SB_OP_LE: case SB_OP_GT: case SB_OP_GE: {
        int64_t b = st[--sp], a = st[sp - 1];
        bool n2 = nl[sp] | nl[sp - 1];
        int c;
        if (nd.arg == SB_VT_F64) c = cmp_f64(__longlong_as_double(a), __longlong_as_double(b));
        else c = a == b ? 0 : (a < b ? -1 : 1);
        bool r = nd.op == SB_OP_EQ ? c == 0 : nd.op == SB_OP_NE ? c != 0 : nd.op == SB_OP_LT ? c < 0
                 : nd.op == SB_OP_LE ? c <= 0 : nd.op == SB_OP_GT ? c > 0 : c >= 0;
        st[sp - 1] = r; nl[sp - 1] = n2;
        break;
      }
      case SB_OP_AND: {
        bool b = st[--sp] != 0, bn = nl[sp], a = st[sp - 1] != 0, an = nl[sp - 1];
        bool is_false = (!an && !a) || (!bn && !b);
        bool is_null = !is_false && (an || bn);
        st[sp - 1] = (!is_false && !is_null) ? 1 : 0; nl[sp - 1] = is_null;
        break;
      }
      case SB_OP_OR: {
        bool b = st[--sp] != 0, bn = nl[sp], a = st[sp - 1] != 0, an = nl[sp - 1];
        bool is_true = (!an && a) || (!bn && b);
        bool is_null = !is_true && (an || bn);
        st[sp - 1] = is_true ? 1 : 0; nl[sp - 1] = is_null;
        break;
      }
      case SB_OP_NOT: st[sp - 1] = st[sp - 1] == 0; break;
      case SB_OP_ISNULL: st[sp - 1] = nl[sp - 1]; nl[sp - 1] = false; break;
      case SB_OP_ISNOTNULL: st[sp - 1] = !nl[sp - 1]; nl[sp - 1] = false; break;
      case SB_OP_CAST_F64:
        if (nd.arg != SB_VT_F64) st[sp - 1] = __double_as_longlong((double)st[sp - 1]);
        break;
      case SB_OP_CAST_I64:
        if (nd.arg == SB_VT_F64) {   // Java (long) d: NaN -> 0, saturating
          double d = __longlong_as_double(st[sp - 1]);
          st[sp - 1] = d != d ? 0 : __double2ll_rz(d);
        }
        break;
      case SB_OP_CAST_I32:
        if (nd.arg == SB_VT_F64) {   // Java (int) d
          double d = __longlong_as_double(st[sp - 1]);
          st[sp - 1] = d != d ? 0 : (int64_t)__double2int_rz(d);
        } else st[sp - 1] = (int64_t)(int32_t)(uint32_t)st[sp - 1];
        break;
      case SB_OP_STR_EQ: case SB_OP_STR_LT: case SB_OP_STR_LE: case SB_OP_STR_GT: case SB_OP_STR_GE: case SB_OP_STR_IN:
      case SB_OP_STR_STARTS_WITH: case SB_OP_STR_ENDS_WITH: case SB_OP_STR_CONTAINS: case SB_OP_STR_LIKE: case SB_OP_STR_OCTET_LENGTH: case SB_OP_STR_CHAR_LENGTH: {
        const int c = nd.arg;
        const bool v = bit_valid(p.col_valid[c], row);
        int64_t x = 0;
        if (v) {
          const int32_t b = p.col_offsets[c][row];
          x = eval_string_test(nd.op, (uint32_t)nd.lit, p.blob, (const uint8_t *)p.col_data[c] + b, p.col_offsets[c][row + 1] - b);
        }
        st[sp] = x; nl[sp] = !v || (nd.op == SB_OP_STR_IN && x == 0 && nd.arg2 != 0); sp++;
        break;
      }
    }
  }
  out = st[0];
  out_null = nl[0];
}

__global__ void __launch_bounds__(256) predicate_kernel(DevProg p, int64_t n, uint8_t *__restrict__ mask) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t v;
  bool nul;
  eval_row(p, i, v, nul);
  mask[i] = (!nul && v != 0) ? 1 : 0;
}

__global__ void __launch_bounds__(256) projection_kernel(DevProg p, const int64_t *__restrict__ sel, int64_t nout, int32_t out_type,
                                                         void *__restrict__ out, uint32_t *__restrict__ out_valid) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool in_range = i < nout;
  int64_t v = 0;
  bool nul = true;
  if (in_range) {
    int64_t row = sel ? sel[i] : i;
    eval_row(p, row, v, nul);
    if (nul) v = 0;
    switch (out_type) {
      case SB_BOOL: ((uint8_t *)out)[i] = v != 0; break;
      case SB_INT8: ((int8_t *)out)[i] = (int8_t)v; break;
      case SB_INT16: ((int16_t *)out)[i] = (int16_t)v; break;
      case SB_INT32: case SB_DATE32: ((int32_t *)out)[i] = (int32_t)v; break;
      case SB_FLOAT32: ((float *)out)[i] = (float)__longlong_as_double(v); break;
      default: ((int64_t *)out)[i] = v; break;
    }
  }
  if (out_valid) {
    uint32_t word = __ballot_sync(0xffffffffu, in_range && !nul);
    if ((threadIdx.x & 31) == 0 && (i - (i & 31)) < nout) out_valid[i >> 5] = word;
  }
}

// ---- fast path: conjunctions of column-vs-literal comparisons (most pushed-down filters: Q1, Q3, Q5, Q6 ...) ----------------
// Same semantics as the interpreter (a comparison with NULL is NULL, a row survives only if every term is TRUE; doubles compare
// like SQLOrderingUtil.compareDoubles), but typed, vectorised and without the per-row program walk: a thread evaluates 16
// consecutive rows from 16-byte loads and stores its 16 mask bytes with one 16-byte store.
bool match_simple_predicate(const sb_table *in, const sb_expr &e, SimplePred &sp) {
  struct Item { int kind; int col; int64_t li; double ld; bool is_f; };   // kind: 0 column, 1 literal, 2 term set
  std::vector<Item> stk;
  sp.nterms = 0;
  auto add_term = [&](const Column &c, int op, int f64, int64_t lit) {
    if (sp.nterms >= SP_MAX_TERMS || c.type == SB_STRING) return false;
    const int i = sp.nterms++;
    sp.type[i] = c.type; sp.op[i] = op; sp.f64[i] = f64; sp.data[i] = c.d(); sp.valid[i] = c.v(); sp.lit[i] = lit;
    return true;
  };
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    if (nd.op == SB_OP_COL) { stk.push_back({0, nd.arg, 0, 0.0, false}); continue; }
    if (nd.op == SB_OP_LIT_I64) { stk.push_back({1, 0, nd.lit.i, (double)nd.lit.i, false}); continue; }
    if (nd.op == SB_OP_LIT_F64) { stk.push_back({1, 0, 0, nd.lit.d, true}); continue; }
    if (nd.op == SB_OP_ISNOTNULL) {
      if (stk.empty() || stk.back().kind != 0) return false;
      const Column &c = in->cols[stk.back().col];
      stk.pop_back();
      if (!add_term(c, SP_NOTNULL, 0, 0)) return false;
      stk.push_back({2, 0, 0, 0.0, false});
      continue;
    }
    if (nd.op == SB_OP_AND) {
      if (stk.size() < 2 || stk.back().kind != 2 || stk[stk.size() - 2].kind != 2) return false;
      stk.pop_back();
      continue;
    }
    if (nd.op >= SB_OP_EQ && nd.op <= SB_OP_GE) {
      if (stk.size() < 2) return false;
      Item r = stk.back(); stk.pop_back();
      Item l = stk.back(); stk.pop_back();
      int op = nd.op - SB_OP_EQ;
      if (l.kind == 1 && r.kind == 0) {   // lit cmp col -> col cmp' lit
        std::swap(l, r);
        static const int flip[6] = {SP_EQ, SP_NE, SP_GT, SP_GE, SP_LT, SP_LE};
        op = flip[op];
      }
      if (l.kind != 0 || r.kind != 1) return false;
      const Column &c = in->cols[l.col];
      if (nd.arg == SB_VT_F64) {
        if (c.type != SB_FLOAT64 && c.type != SB_FLOAT32) return false;
        int64_t bits;
        memcpy(&bits, &r.ld, 8);
        if (!add_term(c, op, 1, bits)) return false;
      } else {
        if (c.type == SB_FLOAT64 || c.type == SB_FLOAT32 || r.is_f) return false;
        if (!add_term(c, op, 0, r.li)) return false;
      }
      stk.push_back({2, 0, 0, 0.0, false});
      continue;
    }
    return false;
  }
  return stk.size() == 1 && stk.back().kind == 2 && sp.nterms >= 1;
}

__global__ void __launch_bounds__(256) simple_predicate_kernel(const __grid_constant__ SimplePred sp, int64_t n, uint8_t *__restrict__ mask) {
  const int64_t row0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * SP_ROWS;
  if (row0 >= n) return;
  const uint32_t keep = simple_pred_eval16(sp, row0, n);
  if (row0 + SP_ROWS <= n) {   // mask + row0 is 16-byte aligned (scratch allocations are)
    uint32_t w[4];
#pragma unroll
    for (int q = 0; q < 4; q++)
      w[q] = ((keep >> (4 * q)) & 1u) | (((keep >> (4 * q + 1)) & 1u) << 8) | (((keep >> (4 * q + 2)) & 1u) << 16) | (((keep >> (4 * q + 3)) & 1u) << 24);
    *reinterpret_cast<uint4 *>(mask + row0) = make_uint4(w[0], w[1], w[2], w[3]);
  } else {
    for (int j = 0; j < SP_ROWS && row0 + j < n; j++) mask[row0 + j] = (keep >> j) & 1u;
  }
}

void eval_predicate(const sb_table *in, const sb_expr &pred, uint8_t *mask, cudaStream_t st) {
  expr_validate(in, pred);   // before the fast path: its matcher trusts the program (a DECIMAL term would compare unscaled values)
  int64_t n = in->nrows;
  if (n == 0) return;
  KernelTimer kt("filter_project", st);
  SimplePred sp;
  const bool no_fast = config().expr_interpret_only != 0;   // parity tests run both paths
  if (!no_fast && ((uintptr_t)mask & 15) == 0 && match_simple_predicate(in, pred, sp)) {
    const int64_t threads = (n + SP_ROWS - 1) / SP_ROWS;
    simple_predicate_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(sp, n, mask);
    SB_LAUNCH_CHECK();
    return;
  }
  const StrTests tests = strpred_compile(pred);
  StrBlob blob(tests, st);
  DevProg p = build_prog(in, pred, tests, blob.ptr());
  predicate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, n, mask);
  SB_LAUNCH_CHECK();
}

Column eval_projection(const sb_table *in, const sb_expr &e, const int64_t *sel, int64_t nout, cudaStream_t st) {
  int col;
  if (expr_is_column(e, &col)) {
    SB_REQUIRE(col >= 0 && col < (int)in->cols.size(), "projection column %d out of range", col);
    if (!sel) return column_share(in->cols[col]);
    return gather_column(in->cols[col], sel, nout, false, st);
  }
  expr_validate(in, e);
  const StrTests tests = strpred_compile(e);
  StrBlob blob(tests, st);
  DevProg p = build_prog(in, e, tests, blob.ptr());
  SB_REQUIRE(e.out_type != SB_STRING && type_width(e.out_type) > 0, "bad projection result type %d", e.out_type);
  Column r = column_alloc(e.out_type, 0, nout, expr_nullable(in, e), st);
  if (nout == 0) return r;
  KernelTimer kt("filter_project", st);
  projection_kernel<<<(unsigned)((nout + 255) / 256), 256, 0, st>>>(p, sel, nout, e.out_type, r.data->ptr,
                                                                    r.validity ? (uint32_t *)r.validity->ptr : nullptr);
  SB_LAUNCH_CHECK();
  return r;
}

}  // namespace sb

using namespace sb;

extern "C" int sb_filter_project(const sb_table *in, const sb_expr *predicate, const sb_expr *projections, int32_t nproj,
                                 sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(in && out && nproj >= 0 && (nproj == 0 || projections), "null argument");
  cudaStream_t st = stream_of(s);
  int64_t n = in->nrows;
  int64_t nout = n;
  Scratch sel(predicate ? n * 8 + 8 : 0, st);
  if (predicate) {
    Scratch mask(n + 16, st);
    eval_predicate(in, *predicate, mask.as<uint8_t>(), st);
    nout = compact_mask(mask.as<uint8_t>(), n, sel.as<int64_t>(), st);
  }
  sb_table *t = table_new(nout);
  try {
    for (int k = 0; k < nproj; k++)
      t->cols.push_back(eval_projection(in, projections[k], predicate ? sel.as<int64_t>() : nullptr, nout, st));
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
  SB_API_END
}

// ---- ExpandExec (SQLX/ExpandExec.scala:36-110): every projection list is evaluated over the whole input (nlists tables of n rows),
// the tables are concatenated and one gather interleaves them so that row r of the input yields output rows r * nlists + l --
// the order of the reference's `iter.flatMap { input => groups.iterator.map(_(input)) }`.
__global__ void interleave_index_kernel(int64_t n, int32_t k, int64_t *__restrict__ idx) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n * k) idx[j] = (j % k) * n + j / k;
}

extern "C" int sb_expand(const sb_table *in, const sb_expr *projections, int32_t nlists, int32_t ncols, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(in && out && projections && nlists >= 1 && ncols >= 1, "bad argument");
  cudaStream_t st = stream_of(s);
  const int64_t n = in->nrows;
  std::vector<sb_table *> parts;
  struct Free {
    std::vector<sb_table *> &v;
    ~Free() { for (auto *t : v) table_free(t); }
  } guard{parts};
  for (int l = 0; l < nlists; l++) {
    sb_table *t = table_new(n);
    parts.push_back(t);
    for (int c = 0; c < ncols; c++) {
      const sb_expr &e = projections[(int64_t)l * ncols + c];
      expr_validate(in, e);
      t->cols.push_back(eval_projection(in, e, nullptr, n, st));
      if (l > 0) SB_REQUIRE(t->cols[c].type == parts[0]->cols[c].type, "expand: column %d has type %d in list %d and %d in list 0", c, t->cols[c].type, l, parts[0]->cols[c].type);
    }
  }
  if (nlists == 1) {
    *out = parts[0];
    parts.clear();
    return SB_OK;
  }
  sb_table *cat = nullptr;
  {
    int rc = sb_table_concat(parts.data(), nlists, s, &cat);
    if (rc != SB_OK) fail(rc, "%s", sb_last_error());
  }
  struct FreeOne { sb_table *t; ~FreeOne() { if (t) table_free(t); } } g2{cat};
  Scratch idx(n * nlists * 8 + 16, st);
  if (n > 0) {
    interleave_index_kernel<<<(unsigned)((n * nlists + 255) / 256), 256, 0, st>>>(n, nlists, idx.as<int64_t>());
    SB_LAUNCH_CHECK();
  }
  *out = gather_table(cat, idx.as<int64_t>(), n * nlists, false, st);
  SB_API_END
}
