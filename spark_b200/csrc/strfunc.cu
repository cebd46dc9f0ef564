// strfunc.cu -- string-producing functions: ProjectExec of SUBSTRING, CONCAT, CONCAT_WS, TRIM / LTRIM / RTRIM and LPAD / RPAD
// (sb_string_project).
//
// Reference semantics restated (no code shared), UTF8_BINARY collation, non-ANSI:
//   Substring   UTF8String.substringSQL: 1-based pos, 0 means 1, a negative pos counts from the end; start + len clamped as a long
//               to the int range; then substring(start, until), which steps code points from the first byte
//   Concat      UTF8String.concat: NULL if any input is NULL
//   ConcatWs    UTF8String.concatWs: NULL inputs are skipped (all of them NULL: the empty string); a NULL separator gives NULL
//   trim()      bytes 0x20 only, from either end
//   trim(set)   trimLeft(set).trimRight(set): a code point goes when its bytes occur anywhere in the set's bytes (UTF8String.find)
//   LPad / RPad len <= 0 gives the empty string; a string at least len code points long, or an empty pad, is cut to len code points;
//               else the pad repeats (its last copy cut to whole code points) in front of / behind the string
// A code point is one step of UTF8String.numBytesForFirstByte (strp_step), so ill-formed bytes step as the reference steps them.
// A truncated lead byte at the end of a value declares more bytes than remain: the trims clamp such a character to the value, as the
// reference does; substring and pad cut at the value's end there too (the reference's copy would run past the value).
//
// Passes (one program = one output column):
//   1. sf_size_kernel, thread per row: the row's value as at most SF_PIECES byte ranges ("pieces") into the input arenas and the
//      literal pool (a pad is one periodic piece); writes the byte length and the validity bit.  Nothing is materialised.
//   2. exclusive scan of the lengths (int64), and ONE stream synchronisation for the arena sizes of all programs of the call; an
//      arena above 2^31 - 1 bytes is refused before any int32 offset is written.
//   3. sf_copy_kernel, thread per row again: the same pieces, then the int32 offsets and the bytes -- a short value by its own
//      thread, a long one by the whole warp (the lanes take turns broadcasting their pieces).
#include <vector>
#include "common.cuh"
#include "strpred.cuh"
#include "primitives.cuh"

namespace sb {

namespace {

constexpr int SF_MAX_NODES = 32;
constexpr int SF_MAX_COLS = 8;
constexpr int SF_PIECES = SB_SF_MAX_RANGES;
constexpr int SF_STACK = SF_PIECES + 1;         // every stack entry may hold a range, so the range cap bounds the depth
constexpr int SF_SHORT = 64;                     // values up to this many bytes are copied by their own thread
constexpr int64_t SF_LEN_CAP = 1ll << 40;        // piece lengths saturate here (16 of them cannot overflow an int64)
constexpr int64_t SF_ROW_CAP = 1ll << 31;        // a row's length saturates here: any row this long fails the arena check on
                                                 // its own, and n rows of it cannot wrap the int64 scan

struct SfNode {
  int32_t op, arg, arg2;
  uint32_t off, len;   // literal slice in the device pool
};
struct SfProg {
  int32_t n;
  SfNode nodes[SF_MAX_NODES];
  const uint8_t *pool;
  const uint8_t *data[SF_MAX_COLS];
  const int32_t *offs[SF_MAX_COLS];
  const uint8_t *valid[SF_MAX_COLS];
};

// a byte range; period != 0: byte k is p[(phase + k) % period] (a repeated pad)
struct Piece {
  const uint8_t *p;
  int64_t len;
  uint32_t period, phase;
};

// ---- host: validation ---------------------------------------------------------------------------------------------------------
void sf_validate(const sb_table *in, const sb_expr &e, int k) {
  SB_REQUIRE(e.nodes && e.n >= 1 && e.n <= SF_MAX_NODES, "string program %d must have 1..%d nodes (got %d)", k, SF_MAX_NODES, e.n);
  SB_REQUIRE(e.out_type == SB_STRING, "string program %d: out_type %d is not STRING", k, e.out_type);
  SB_REQUIRE(e.nbytes >= 0 && (e.nbytes == 0 || e.bytes), "string program %d: bad literal pool", k);
  int pieces[SF_STACK + 1];   // ranges each stack entry may hold
  int depth = 0, total = 0;
  int cols[SF_MAX_COLS], ncols = 0;
  auto slice_ok = [&](const sb_expr_node &nd) {
    const uint64_t off = (uint64_t)nd.lit.i >> 32, len = (uint64_t)nd.lit.i & 0xffffffffu;
    return off + len <= (uint64_t)e.nbytes;
  };
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    SB_REQUIRE(nd.vtype == 0, "string program %d node %d: vtype %d, expected 0", k, i, nd.vtype);
    int pops = 0, res = 0;
    switch (nd.op) {
      case SB_OP_SF_COL: {
        SB_REQUIRE(nd.arg >= 0 && nd.arg < (int)in->cols.size(), "string program %d node %d references column %d of %zu", k, i, nd.arg,
                   in->cols.size());
        SB_REQUIRE(in->cols[nd.arg].type == SB_STRING, "string program %d node %d: column %d has type %d, not STRING", k, i, nd.arg,
                   in->cols[nd.arg].type);
        SB_REQUIRE(nd.arg2 == 0 && nd.lit.i == 0, "string program %d node %d: SF_COL takes no literal", k, i);
        bool seen = false;
        for (int c = 0; c < ncols; c++) seen |= cols[c] == nd.arg;
        if (!seen) {
          SB_REQUIRE(ncols < SF_MAX_COLS, "string program %d references more than %d distinct columns", k, SF_MAX_COLS);
          cols[ncols++] = nd.arg;
        }
        res = 1;
        break;
      }
      case SB_OP_SF_LIT:
        SB_REQUIRE(nd.arg == 0 && (nd.arg2 == 0 || nd.arg2 == 1) && slice_ok(nd), "string program %d node %d: bad SF_LIT", k, i);
        res = 1;
        break;
      case SB_OP_SF_SUBSTRING:
        pops = 1;
        SB_REQUIRE(depth >= 1, "string program %d: stack underflow at node %d", k, i);
        res = pieces[depth - 1];
        break;
      case SB_OP_SF_TRIM: case SB_OP_SF_LTRIM: case SB_OP_SF_RTRIM:
        pops = 1;
        SB_REQUIRE(depth >= 1, "string program %d: stack underflow at node %d", k, i);
        SB_REQUIRE((nd.arg == 0 || nd.arg == 1) && nd.arg2 == 0 && slice_ok(nd) && (nd.arg == 1 || nd.lit.i == 0),
                   "string program %d node %d: bad trim (arg %d)", k, i, nd.arg);
        res = pieces[depth - 1];
        break;
      case SB_OP_SF_LPAD: case SB_OP_SF_RPAD:
        pops = 1;
        SB_REQUIRE(depth >= 1, "string program %d: stack underflow at node %d", k, i);
        SB_REQUIRE(nd.arg2 == 0 && slice_ok(nd), "string program %d node %d: bad pad", k, i);
        res = pieces[depth - 1] + 1;
        break;
      case SB_OP_SF_CONCAT: case SB_OP_SF_CONCAT_WS:
        pops = nd.arg;
        SB_REQUIRE(nd.arg >= 1 && nd.arg <= depth, "string program %d node %d: concatenates %d of %d stack values", k, i, nd.arg, depth);
        SB_REQUIRE(nd.arg2 == 0 && slice_ok(nd) && (nd.op == SB_OP_SF_CONCAT_WS || nd.lit.i == 0), "string program %d node %d: bad concat", k, i);
        for (int j = 0; j < nd.arg; j++) res += pieces[depth - 1 - j];
        if (nd.op == SB_OP_SF_CONCAT_WS) res += nd.arg - 1;
        break;
      default: fail(SB_ERR_INVALID, "string program %d: unknown op %d at node %d", k, nd.op, i);
    }
    for (int j = 0; j < pops; j++) total -= pieces[--depth];
    total += res;
    if (total > SF_PIECES)
      fail(SB_ERR_UNSUPPORTED, "string program %d: node %d needs %d byte ranges, more than the %d a value is assembled from", k, i, total, SF_PIECES);
    pieces[depth++] = res;   // depth <= total < SF_STACK: every entry counts at least one range
  }
  SB_REQUIRE(depth == 1, "string program %d leaves %d values on the stack", k, depth);
}

bool sf_nullable(const sb_table *in, const sb_expr &e) {
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    if (nd.op == SB_OP_SF_COL && in->cols[nd.arg].validity) return true;
    if (nd.op == SB_OP_SF_LIT && nd.arg2) return true;
  }
  return false;
}

SfProg sf_build(const sb_table *in, const sb_expr &e, const uint8_t *pool_dev) {
  SfProg p;
  memset(&p, 0, sizeof(p));
  p.n = e.n;
  p.pool = pool_dev;
  std::vector<int> remap;
  int ncols = 0;
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    SfNode &d = p.nodes[i];
    d.op = nd.op;
    d.arg = nd.arg;
    d.arg2 = nd.arg2;
    d.off = (uint32_t)((uint64_t)nd.lit.i >> 32);
    d.len = (uint32_t)((uint64_t)nd.lit.i & 0xffffffffu);
    if (nd.op == SB_OP_SF_COL) {
      int c = -1;
      for (size_t j = 0; j < remap.size(); j++)
        if (remap[j] == nd.arg) c = (int)j;
      if (c < 0) {
        c = ncols++;
        remap.push_back(nd.arg);
        const Column &col = in->cols[nd.arg];
        p.data[c] = (const uint8_t *)col.d();
        p.offs[c] = col.o();
        p.valid[c] = col.v();
      }
      d.arg = c;
    }
  }
  return p;
}

// ---- device: evaluation -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t piece_byte(const Piece &q, int64_t k) {
  return q.period ? q.p[(q.phase + (uint64_t)k) % q.period] : q.p[k];
}

// the byte at logical position `at` of pieces [b, e) (at is inside them)
__device__ uint8_t entry_byte(const Piece *pc, int b, int e, int64_t at) {
  for (int i = b; i < e; i++) {
    if (at < pc[i].len) return piece_byte(pc[i], at);
    at -= pc[i].len;
  }
  return 0;
}

// reads forward through pieces [b, e) from logical position 0
struct Cursor {
  const Piece *pc;
  int i, e;
  int64_t off;   // inside piece i
  int64_t pos;   // logical
  __device__ Cursor(const Piece *pc_, int b, int e_) : pc(pc_), i(b), e(e_), off(0), pos(0) { settle(); }
  __device__ void settle() {
    while (i < e && off >= pc[i].len) {
      off -= pc[i].len;
      i++;
    }
  }
  __device__ uint8_t byte() const { return piece_byte(pc[i], off); }
  __device__ void skip(int64_t k) {
    off += k;
    pos += k;
    settle();
  }
};

// logical end of pieces [b, e)
__device__ __forceinline__ int64_t entry_len(const Piece *pc, int b, int e) {
  int64_t t = 0;
  for (int i = b; i < e; i++) t += pc[i].len;
  return t;
}

// position after `count` code points from `c` (never past total), and how many were stepped
__device__ int64_t step_chars(Cursor &c, int64_t total, int64_t count, int64_t *stepped) {
  int64_t n = 0;
  while (c.pos < total && n < count) {
    c.skip(strp_step(c.byte()));
    n++;
  }
  if (stepped) *stepped = n;
  return c.pos;
}

// keeps logical bytes [a, z) of pieces [b, *e); a <= z <= length
__device__ void slice_entry(Piece *pc, int b, int *e, int64_t a, int64_t z) {
  int w = b;
  int64_t at = 0;
  for (int i = b; i < *e; i++) {
    const Piece q = pc[i];
    const int64_t lo = at > a ? at : a, hi = at + q.len < z ? at + q.len : z;
    if (hi > lo) {
      Piece r = q;
      const int64_t cut = lo - at;
      if (q.period) r.phase = (uint32_t)((q.phase + (uint64_t)cut) % q.period);
      else r.p = q.p + cut;
      r.len = hi - lo;
      pc[w++] = r;
    }
    at += q.len;
  }
  *e = w;
}

// does the character c[0..w) occur in the literal l[0..m) (UTF8String.find from 0)?
__device__ bool in_set(const uint8_t *c, int w, const uint8_t *l, uint32_t m) {
  for (int64_t s = 0; s + w <= (int64_t)m; s++) {
    bool eq = true;
    for (int k = 0; k < w && eq; k++) eq = l[s + k] == c[k];
    if (eq) return true;
  }
  return false;
}

// the character at the cursor, clamped to the value (copyUTF8String); returns its width
__device__ int read_char(Cursor &c, int64_t total, uint8_t ch[4]) {
  const int64_t start = c.pos;
  const int w = strp_step(c.byte());
  const int wc = (int)(start + w <= total ? w : total - start);
  for (int k = 0; k < wc; k++) {
    ch[k] = c.byte();
    c.skip(1);
  }
  return wc;
}

// the value of program p for `row`: pieces pc[0..*np), and whether it is NULL
__device__ __forceinline__ bool sf_eval(const SfProg &p, int64_t row, Piece *pc, int *np_out) {
  int base[SF_STACK];
  bool nul[SF_STACK];
  int sp = 0, np = 0;
#pragma unroll 1
  for (int k = 0; k < p.n; k++) {
    const SfNode nd = p.nodes[k];
    switch (nd.op) {
      case SB_OP_SF_COL: {
        const int c = nd.arg;
        base[sp] = np;
        nul[sp] = !bit_valid(p.valid[c], row);
        if (!nul[sp]) {
          const int32_t o = p.offs[c][row];
          pc[np++] = Piece{p.data[c] + o, (int64_t)(p.offs[c][row + 1] - o), 0u, 0u};
        }
        sp++;
        break;
      }
      case SB_OP_SF_LIT:
        base[sp] = np;
        nul[sp] = nd.arg2 != 0;
        if (!nul[sp]) pc[np++] = Piece{p.pool + nd.off, (int64_t)nd.len, 0u, 0u};
        sp++;
        break;
      case SB_OP_SF_CONCAT: {
        const int first = sp - nd.arg;
        bool any = false;
        for (int j = first; j < sp; j++) any |= nul[j];
        sp = first + 1;
        nul[first] = any;
        if (any) np = base[first];
        break;
      }
      case SB_OP_SF_CONCAT_WS: {
        // move the operands' pieces to the top of the array, then write them back with separators between the non-NULL ones
        const int first = sp - nd.arg, b = base[first], m = np - b;
        int ends[SF_STACK];
        for (int j = first; j < sp; j++) ends[j] = j + 1 < sp ? base[j + 1] : np;
        for (int t = m - 1; t >= 0; t--) pc[SF_PIECES - m + t] = pc[b + t];
        const int shift = SF_PIECES - m - b;
        int w = b;
        bool seen = false;
        for (int j = first; j < sp; j++) {
          if (nul[j]) continue;
          if (seen) pc[w++] = Piece{p.pool + nd.off, (int64_t)nd.len, 0u, 0u};
          seen = true;
          for (int t = base[j] + shift; t < ends[j] + shift; t++) pc[w++] = pc[t];
        }
        np = w;
        sp = first + 1;
        nul[first] = false;
        break;
      }
      default: {   // unary: the top entry
        const int b = base[sp - 1];
        if (nul[sp - 1]) break;
        const int64_t total = entry_len(pc, b, np);
        if (nd.op == SB_OP_SF_SUBSTRING) {
          const int32_t pos = nd.arg, len = nd.arg2;
          int64_t start = 0;
          if (pos > 0) start = pos - 1;
          else if (pos < 0) {
            Cursor c(pc, b, np);
            int64_t chars;
            step_chars(c, total, INT64_MAX, &chars);
            start = chars + pos;   // int in the reference: numChars() + pos cannot overflow (numChars >= 0 > pos)
          }
          int64_t until = start + len;
          if (until > INT32_MAX) until = INT32_MAX;
          if (until < INT32_MIN) until = INT32_MIN;
          if (until <= start || start >= total) {
            np = b;
            break;
          }
          // UTF8String.substring(start, until): step `start` code points (none when start < 0), then on to code point `until`
          const int64_t first = start < 0 ? 0 : start;
          Cursor c(pc, b, np);
          const int64_t j = step_chars(c, total, first, nullptr);
          const int64_t i = until == INT32_MAX ? total : step_chars(c, total, until - first, nullptr);
          slice_entry(pc, b, &np, j, i);
        } else if (nd.op == SB_OP_SF_TRIM || nd.op == SB_OP_SF_LTRIM || nd.op == SB_OP_SF_RTRIM) {
          const bool left = nd.op != SB_OP_SF_RTRIM, right = nd.op != SB_OP_SF_LTRIM;
          int64_t s = 0, z = total;
          if (nd.arg == 0) {   // trim(): bytes 0x20
            if (left) {
              Cursor c(pc, b, np);
              while (c.pos < total && c.byte() == 0x20) c.skip(1);
              s = c.pos;
            }
            if (right)
              while (z > s && entry_byte(pc, b, np, z - 1) == 0x20) z--;
          } else {
            const uint8_t *set = p.pool + nd.off;
            Cursor c(pc, b, np);
            uint8_t ch[4];
            if (left) {
              while (c.pos < total) {
                const int64_t at = c.pos;
                const int w = read_char(c, total, ch);
                if (!in_set(ch, w, set, nd.len)) {
                  s = at;
                  break;
                }
                s = c.pos;
              }
              c = Cursor(pc, b, np);
              c.skip(s);
            }
            if (right) {   // the end of the last character that is not in the set
              z = s;
              while (c.pos < total) {
                const int w = read_char(c, total, ch);
                if (!in_set(ch, w, set, nd.len)) z = c.pos;
              }
            }
          }
          slice_entry(pc, b, &np, s, z);
        } else {   // LPAD / RPAD
          const int32_t len = nd.arg;
          if (len <= 0) {
            np = b;
            break;
          }
          Cursor c(pc, b, np);
          int64_t chars;
          step_chars(c, total, INT64_MAX, &chars);
          const int64_t spaces = (int64_t)len - chars;
          if (spaces <= 0 || nd.len == 0) {
            Cursor c2(pc, b, np);
            slice_entry(pc, b, &np, 0, step_chars(c2, total, len, nullptr));
            break;
          }
          const uint8_t *pad = p.pool + nd.off;
          int64_t pad_chars = 0;
          for (uint32_t i = 0; i < nd.len; i += strp_step(pad[i])) pad_chars++;
          const int64_t count = spaces / pad_chars, rem = spaces - pad_chars * count;
          uint32_t rem_bytes = 0;
          for (int64_t r = 0; r < rem && rem_bytes < nd.len; r++) rem_bytes += strp_step(pad[rem_bytes]);
          if (rem_bytes > nd.len) rem_bytes = nd.len;
          int64_t plen = count * (int64_t)nd.len + rem_bytes;
          if (plen > SF_LEN_CAP) plen = SF_LEN_CAP;
          const Piece q{pad, plen, nd.len, 0u};
          if (nd.op == SB_OP_SF_RPAD) {
            pc[np++] = q;
          } else {
            for (int t = np; t > b; t--) pc[t] = pc[t - 1];
            pc[b] = q;
            np++;
          }
        }
        break;
      }
    }
  }
  *np_out = nul[0] ? 0 : np;
  return nul[0];
}

__global__ void __launch_bounds__(256, 1) sf_size_kernel(const __grid_constant__ SfProg p, int64_t n, int64_t *__restrict__ lens,
                                                      uint32_t *__restrict__ out_valid) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in_range = row < n;
  bool nul = true;
  if (in_range) {
    Piece pc[SF_PIECES];
    int np;
    nul = sf_eval(p, row, pc, &np);
    int64_t t = 0;
    for (int i = 0; i < np; i++) t += pc[i].len < SF_LEN_CAP ? pc[i].len : SF_LEN_CAP;
    lens[row] = t < SF_ROW_CAP ? t : SF_ROW_CAP;
  }
  if (out_valid) {
    const uint32_t word = __ballot_sync(0xffffffffu, in_range && !nul);
    if ((threadIdx.x & 31) == 0 && (row - (row & 31)) < n) out_valid[row >> 5] = word;
  }
}

__global__ void __launch_bounds__(256, 1) sf_copy_kernel(const __grid_constant__ SfProg p, int64_t n, const int64_t *__restrict__ off64,
                                                      int32_t *__restrict__ out_off, uint8_t *__restrict__ arena) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool in_range = row < n;
  Piece pc[SF_PIECES];
  int np = 0;
  int64_t off = 0, len = 0;
  if (in_range) {
    sf_eval(p, row, pc, &np);
    for (int i = 0; i < np; i++) len += pc[i].len;
    off = off64[row];
    out_off[row] = (int32_t)off;
    if (row == n - 1) out_off[n] = (int32_t)(off + len);
  }
  const bool longv = len > SF_SHORT;
  if (in_range && !longv) {
    uint8_t *d = arena + off;
    for (int i = 0; i < np; i++) {
      const Piece q = pc[i];
      if (!q.period) {
        for (int64_t k = 0; k < q.len; k++) d[k] = q.p[k];
      } else {
        uint32_t ix = q.phase;
        for (int64_t k = 0; k < q.len; k++) {
          d[k] = q.p[ix];
          if (++ix == q.period) ix = 0;
        }
      }
      d += q.len;
    }
  }
  // long values: the warp copies them one at a time, their owner broadcasting each piece
  uint32_t todo = __ballot_sync(0xffffffffu, in_range && longv);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const int kn = __shfl_sync(0xffffffffu, np, src);
    int64_t at = __shfl_sync(0xffffffffu, off, src);
    for (int i = 0; i < kn; i++) {
      const Piece mine = pc[i < SF_PIECES ? i : 0];
      const uint8_t *qp = (const uint8_t *)__shfl_sync(0xffffffffu, (unsigned long long)mine.p, src);
      const int64_t qlen = __shfl_sync(0xffffffffu, mine.len, src);
      const uint32_t period = __shfl_sync(0xffffffffu, mine.period, src), phase = __shfl_sync(0xffffffffu, mine.phase, src);
      uint8_t *d = arena + at;
      if (!period) {
        for (int64_t k = lane; k < qlen; k += 32 * 4) {
          uint8_t v[4];
#pragma unroll
          for (int u = 0; u < 4; u++) v[u] = k + 32 * u < qlen ? qp[k + 32 * u] : 0;
#pragma unroll
          for (int u = 0; u < 4; u++)
            if (k + 32 * u < qlen) d[k + 32 * u] = v[u];
        }
      } else {
        uint32_t ix = (uint32_t)((phase + (uint64_t)lane) % period);
        const uint32_t adv = 32 % period;
        for (int64_t k = lane; k < qlen; k += 32) {
          d[k] = qp[ix];
          ix += adv;
          if (ix >= period) ix -= period;
        }
      }
      at += qlen;
    }
  }
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" int sb_string_project(const sb_table *in, const sb_expr *programs, int32_t nprog, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(in && out && nprog >= 0 && (nprog == 0 || programs), "null argument");
  for (int k = 0; k < nprog; k++) sf_validate(in, programs[k], k);
  cudaStream_t st = stream_of(s);
  const int64_t n = in->nrows;
  sb_table *t = table_new(n);
  try {
    std::vector<Scratch *> pools;
    struct FreePools {
      std::vector<Scratch *> &v;
      ~FreePools() { for (auto *p : v) delete p; }
    } guard{pools};
    std::vector<SfProg> progs;
    // per program: the row lengths, scanned in place into the offsets (8 bytes per row and program, all alive until the copies)
    Scratch offs((int64_t)nprog * n * 8 + 16, st), totals((int64_t)nprog * 8 + 16, st);
    const unsigned grid = (unsigned)((n + 255) / 256);
    for (int k = 0; k < nprog; k++) {
      const sb_expr &e = programs[k];
      pools.push_back(new Scratch(e.nbytes + 16, st));
      // pageable source: the copy has read the host bytes when the call returns
      if (e.nbytes) SB_CUDA(cudaMemcpyAsync(pools.back()->ptr, e.bytes, (size_t)e.nbytes, cudaMemcpyHostToDevice, st));
      progs.push_back(sf_build(in, e, pools.back()->as<const uint8_t>()));
      Column c;
      c.type = SB_STRING;
      c.length = n;
      c.null_count = sf_nullable(in, e) ? -1 : 0;
      c.offsets = buffer_alloc((n + 1) * 4 + 16, st);
      if (c.null_count) c.validity = buffer_alloc(bitmap_alloc_bytes(n), st);
      t->cols.push_back(c);
      if (n == 0) continue;
      KernelTimer kt("string_project", st);
      sf_size_kernel<<<grid, 256, 0, st>>>(progs[k], n, offs.as<int64_t>() + (int64_t)k * n,
                                           c.validity ? (uint32_t *)c.validity->ptr : nullptr);
      SB_LAUNCH_CHECK();
      exclusive_scan_i64(offs.as<int64_t>() + (int64_t)k * n, offs.as<int64_t>() + (int64_t)k * n, n, totals.as<int64_t>() + k, st);
    }
    std::vector<int64_t> tot(nprog, 0);
    if (n > 0 && nprog > 0) {
      SB_CUDA(cudaMemcpyAsync(tot.data(), totals.ptr, (size_t)nprog * 8, cudaMemcpyDeviceToHost, st));
      SB_CUDA(cudaStreamSynchronize(st));
    }
    for (int k = 0; k < nprog; k++)
      if (tot[k] > 0x7fffffffll || tot[k] < 0)
        fail(SB_ERR_UNSUPPORTED, "string_project: output %d takes %lld bytes, more than the 2^31 - 1 an int32-offset string column holds", k,
             (long long)tot[k]);
    for (int k = 0; k < nprog; k++) {
      Column &c = t->cols[k];
      c.data = buffer_alloc(tot[k] + 16, st);
      c.string_bytes = tot[k];
      if (n == 0) {
        SB_CUDA(cudaMemsetAsync(c.offsets->ptr, 0, 4, st));
        continue;
      }
      KernelTimer kt("string_project", st);
      sf_copy_kernel<<<grid, 256, 0, st>>>(progs[k], n, offs.as<int64_t>() + (int64_t)k * n, (int32_t *)c.offsets->ptr,
                                           (uint8_t *)c.data->ptr);
      SB_LAUNCH_CHECK();
    }
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
  SB_API_END
}
