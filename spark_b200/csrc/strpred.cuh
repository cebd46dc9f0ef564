// strpred.cuh -- string tests against literals (SB_OP_STR_*): the one module that knows their format.
//
// Reference semantics restated (no code shared), UTF8_BINARY collation:
//   comparisons        UTF8String.binaryCompare: unsigned bytes, a proper prefix first
//   IN / InSet         predicates.scala In.eval / InSet.eval: TRUE on a match, else NULL when the list holds NULL, else FALSE
//   StartsWith / EndsWith / Contains   stringExpressions.scala: byte matching; an empty literal matches every non-NULL string
//   LIKE               regexpExpressions.scala Like + StringUtils.escapeLikeRegex: the whole string matches, `%` = any run of code
//                      points (newlines too), `_` = one code point, the escape character precedes `%`, `_` or itself only
//   octet_length       the byte length
//   length             UTF8String.numChars: one per step, a step being the width its lead byte declares (numBytesForFirstByte)
//
// The host compiles a program's literals into one blob of 32-bit words that is copied to the device once per evaluation; a node's
// test is the word index `ref` of its descriptor in that blob:
//   STR_EQ .. STR_CONTAINS   [length][bytes, padded to a word]
//   STR_IN                   [count][byte offset, length] * count, sorted by binaryCompare, no duplicates (binary search)
//   STR_LIKE                 [nseg][has_percent][unit byte offset, nunits] * nseg; a unit is a uint16: 0..255 a literal byte,
//                            STRP_ANY one code point.  Without `%` the one segment must span the string; with it, segment 0 is
//                            anchored at the start, the last at the end, and every middle one takes its leftmost match.  A
//                            segment matches a fixed number of code points, so where it ends grows with where it starts and the
//                            leftmost match is never worse than a later one: the greedy walk is exact.
// The device matchers take a byte pointer and a length.  A code point starts at a string's first byte and at every later byte that
// is not 10xxxxxx (strings are assumed to be valid UTF-8; DESIGN §2).
#pragma once
#include "common.cuh"

namespace sb {

constexpr uint16_t STRP_ANY = 256;

inline bool strpred_is_leaf(int32_t op) { return op >= SB_OP_STR_EQ && op <= SB_OP_STR_CHAR_LENGTH; }
// the leaves whose value is an I32 length and that take no literal
inline bool strpred_is_length(int32_t op) { return op == SB_OP_STR_OCTET_LENGTH || op == SB_OP_STR_CHAR_LENGTH; }

// host: checks string-test node `i` of `e` against `in` (a string column, the slice inside the pool, a well-formed IN list, the
// LIKE escape rules) and returns the node's value class; SB_ERR_INVALID otherwise
int32_t strpred_validate(const sb_table *in, const sb_expr &e, int i);

// host: the blob of a validated program; ref[i] is node i's descriptor (0 for other nodes)
struct StrTests {
  std::vector<uint32_t> words;
  std::vector<uint32_t> ref;
};
StrTests strpred_compile(const sb_expr &e);

// the blob on the device, stream-ordered (freed in `st`'s order when this goes out of scope)
struct StrBlob {
  Scratch dev;
  StrBlob(const StrTests &t, cudaStream_t st);
  const uint32_t *ptr() { return dev.as<const uint32_t>(); }
};

#ifdef __CUDACC__
__device__ __forceinline__ int strp_compare(const uint8_t *s, int32_t n, const uint8_t *l, int32_t m) {
  const int32_t k = n < m ? n : m;
  for (int32_t i = 0; i < k; i++)
    if (s[i] != l[i]) return (int)s[i] - (int)l[i];
  return n == m ? 0 : (n < m ? -1 : 1);
}

__device__ __forceinline__ bool strp_equal(const uint8_t *s, const uint8_t *l, int32_t m) {
  for (int32_t i = 0; i < m; i++)
    if (s[i] != l[i]) return false;
  return true;
}

__device__ __forceinline__ bool strp_is_cont(uint8_t b) { return (b & 0xC0) == 0x80; }

// UTF8String.numBytesForFirstByte: the width a lead byte declares; 1 for continuation bytes, 0xC0 / 0xC1 and 0xF5..0xFF
__device__ __forceinline__ int strp_step(uint8_t b) { return b < 0xC2 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : b < 0xF5 ? 4 : 1; }

// UTF8String.numChars of s[0..n)
__device__ __forceinline__ int32_t strp_num_chars(const uint8_t *s, int32_t n) {
  int32_t c = 0;
  for (int32_t i = 0; i < n; i += strp_step(s[i])) c++;
  return c;
}

// segment `u[0..k)` forward from p, never past n; p becomes its end
__device__ __forceinline__ bool strp_seg_fwd(const uint16_t *u, int32_t k, const uint8_t *s, int32_t n, int32_t &p) {
  for (int32_t i = 0; i < k; i++) {
    if (p >= n) return false;
    const uint16_t c = u[i];
    if (c != STRP_ANY) {
      if (s[p] != c) return false;
      p++;
    } else {
      p++;
      while (p < n && strp_is_cont(s[p])) p++;
    }
  }
  return true;
}

// segment `u[0..k)` backward from q, never before lo; q becomes its start
__device__ __forceinline__ bool strp_seg_bwd(const uint16_t *u, int32_t k, const uint8_t *s, int32_t lo, int32_t &q) {
  for (int32_t i = k - 1; i >= 0; i--) {
    if (q <= lo) return false;
    const uint16_t c = u[i];
    q--;
    if (c != STRP_ANY) {
      if (s[q] != c) return false;
    } else {
      while (q > lo && strp_is_cont(s[q])) q--;
    }
  }
  return true;
}

__device__ __forceinline__ bool strp_like(const uint32_t *d, const uint8_t *blob, const uint8_t *s, int32_t n) {
  const int32_t nseg = (int32_t)d[0];
  const bool pct = d[1] != 0;
  auto seg = [&](int i) { return (const uint16_t *)(blob + d[2 + 2 * i]); };
  auto len = [&](int i) { return (int32_t)d[3 + 2 * i]; };
  int32_t p = 0;
  if (!strp_seg_fwd(seg(0), len(0), s, n, p)) return false;
  if (!pct) return p == n;
  int32_t q = n;
  if (!strp_seg_bwd(seg(nseg - 1), len(nseg - 1), s, p, q)) return false;
  for (int i = 1; i < nseg - 1; i++) {
    bool found = false;
    for (int32_t st = p; st <= q && !found; st++) {
      if (st > p && st < q && strp_is_cont(s[st])) continue;   // `%` consumes whole code points
      int32_t e = st;
      if (strp_seg_fwd(seg(i), len(i), s, q, e)) {
        p = e;
        found = true;
      }
    }
    if (!found) return false;
  }
  return true;
}

// the value of string test `op` (descriptor `ref`) for the non-NULL string s[0..n): 0 / 1, or the length.  For STR_IN, 0 means
// "no match" (NULL when the list holds NULL: the caller's business).
__device__ __forceinline__ int64_t strpred_eval(int32_t op, uint32_t ref, const uint32_t *__restrict__ blob, const uint8_t *s, int32_t n) {
  const uint32_t *d = blob + ref;
  const uint8_t *b = (const uint8_t *)blob;
  switch (op) {
    case SB_OP_STR_OCTET_LENGTH: return n;
    case SB_OP_STR_CHAR_LENGTH: return strp_num_chars(s, n);
    case SB_OP_STR_IN: {
      int32_t lo = 0, hi = (int32_t)d[0] - 1;
      while (lo <= hi) {
        const int32_t mid = (lo + hi) >> 1;
        const int c = strp_compare(s, n, b + d[1 + 2 * mid], (int32_t)d[2 + 2 * mid]);
        if (c == 0) return 1;
        if (c < 0) hi = mid - 1;
        else lo = mid + 1;
      }
      return 0;
    }
    case SB_OP_STR_LIKE: return strp_like(d, b, s, n);
    default: break;
  }
  const int32_t m = (int32_t)d[0];
  const uint8_t *l = (const uint8_t *)(d + 1);
  switch (op) {
    case SB_OP_STR_STARTS_WITH: return n >= m && strp_equal(s, l, m);
    case SB_OP_STR_ENDS_WITH: return n >= m && strp_equal(s + (n - m), l, m);
    case SB_OP_STR_CONTAINS:
      for (int32_t i = 0; i + m <= n; i++)
        if (strp_equal(s + i, l, m)) return 1;
      return 0;
    case SB_OP_STR_EQ: return n == m && strp_equal(s, l, m);
    default: {
      const int c = strp_compare(s, n, l, m);
      return op == SB_OP_STR_LT ? c < 0 : op == SB_OP_STR_LE ? c <= 0 : op == SB_OP_STR_GT ? c > 0 : c >= 0;
    }
  }
}
#endif

}  // namespace sb
