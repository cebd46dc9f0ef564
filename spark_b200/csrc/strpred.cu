// strpred.cu -- host side of the string tests: validation, the LIKE compiler, sorted IN lists.
// The format and the matchers: strpred.cuh.
#include <algorithm>
#include "strpred.cuh"

namespace sb {

namespace {

struct Slice {
  const uint8_t *p;
  uint32_t len;
};

Slice slice_of(const sb_expr &e, const sb_expr_node &nd) {
  const uint64_t off = (uint64_t)nd.lit.i >> 32, len = (uint64_t)nd.lit.i & 0xffffffffu;
  return {len ? e.bytes + off : nullptr, (uint32_t)len};
}

uint32_t rd32(const uint8_t *p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}

// the records of an IN slice; false when the slice is not exactly [count][length][bytes]*count
bool in_records(Slice s, std::vector<Slice> *out) {
  if (s.len < 4) return false;
  const uint32_t count = rd32(s.p);
  uint64_t pos = 4;
  for (uint32_t k = 0; k < count; k++) {
    if (pos + 4 > s.len) return false;
    const uint32_t l = rd32(s.p + pos);
    pos += 4;
    if (pos + l > s.len) return false;
    if (out) out->push_back({s.p + pos, l});
    pos += l;
  }
  return pos == s.len;
}

// one UTF-8 code point at p[0..n): its value and byte length, or -1 when the bytes are not well-formed UTF-8
int32_t decode_utf8(const uint8_t *p, uint32_t n, int *nb) {
  const uint8_t b = p[0];
  int len;
  int32_t cp;
  if (b < 0x80) { *nb = 1; return b; }
  if ((b & 0xE0) == 0xC0) { len = 2; cp = b & 0x1F; }
  else if ((b & 0xF0) == 0xE0) { len = 3; cp = b & 0x0F; }
  else if ((b & 0xF8) == 0xF0) { len = 4; cp = b & 0x07; }
  else return -1;
  if ((uint32_t)len > n) return -1;
  for (int i = 1; i < len; i++) {
    if ((p[i] & 0xC0) != 0x80) return -1;
    cp = (cp << 6) | (p[i] & 0x3F);
  }
  static const int32_t min_of[5] = {0, 0, 0x80, 0x800, 0x10000};
  if (cp < min_of[len] || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return -1;
  *nb = len;
  return cp;
}

// StringUtils.escapeLikeRegex, as segments of units (strpred.cuh); fails with SB_ERR_INVALID on the reference's two errors
std::vector<std::vector<uint16_t>> like_segments(Slice s, int32_t escape, int node) {
  std::vector<std::vector<uint16_t>> segs(1);
  uint32_t i = 0;
  auto literal = [&](uint32_t at, int nb) {
    for (int k = 0; k < nb; k++) segs.back().push_back(s.p[at + k]);
  };
  while (i < s.len) {
    int nb;
    const int32_t c = decode_utf8(s.p + i, s.len - i, &nb);
    SB_REQUIRE(c >= 0, "STR_LIKE node %d: the pattern is not valid UTF-8 at byte %u", node, i);
    if (c == escape) {
      SB_REQUIRE(i + nb < s.len, "STR_LIKE node %d: the pattern must not end with the escape character", node);
      int nb2;
      const int32_t c2 = decode_utf8(s.p + i + nb, s.len - i - nb, &nb2);
      SB_REQUIRE(c2 >= 0, "STR_LIKE node %d: the pattern is not valid UTF-8 at byte %u", node, i + nb);
      SB_REQUIRE(c2 == '%' || c2 == '_' || c2 == escape, "STR_LIKE node %d: the escape character is not allowed to precede code point %d",
                 node, c2);
      literal(i + nb, nb2);
      i += nb + nb2;
      continue;
    }
    if (c == '%') segs.emplace_back();
    else if (c == '_') segs.back().push_back(STRP_ANY);
    else literal(i, nb);
    i += nb;
  }
  return segs;
}

bool binary_less(const Slice &a, const Slice &b) {
  const uint32_t k = std::min(a.len, b.len);
  const int c = k ? memcmp(a.p, b.p, k) : 0;   // memcmp compares as unsigned char
  return c != 0 ? c < 0 : a.len < b.len;
}

}  // namespace

int32_t strpred_validate(const sb_table *in, const sb_expr &e, int i) {
  const sb_expr_node &nd = e.nodes[i];
  SB_REQUIRE(nd.arg >= 0 && nd.arg < (int)in->cols.size(), "string test node %d references column %d of %zu", i, nd.arg, in->cols.size());
  SB_REQUIRE(in->cols[nd.arg].type == SB_STRING, "string test node %d: column %d has type %d, not STRING", i, nd.arg, in->cols[nd.arg].type);
  const int32_t want = strpred_is_length(nd.op) ? SB_VT_I32 : SB_VT_BOOL;
  SB_REQUIRE(nd.vtype == want, "string test node %d (op %d): vtype %d, expected %d", i, nd.op, nd.vtype, want);
  const uint64_t off = (uint64_t)nd.lit.i >> 32, len = (uint64_t)nd.lit.i & 0xffffffffu;
  SB_REQUIRE(e.nbytes >= 0 && off + len <= (uint64_t)e.nbytes && (len == 0 || e.bytes), "string test node %d: literal [%llu, +%llu) lies outside the %lld pool bytes",
             i, (unsigned long long)off, (unsigned long long)len, (long long)e.nbytes);
  const Slice s = slice_of(e, nd);
  switch (nd.op) {
    case SB_OP_STR_IN:
      SB_REQUIRE(nd.arg2 == 0 || nd.arg2 == 1, "STR_IN node %d: arg2 %d is not 0 or 1", i, nd.arg2);
      SB_REQUIRE(in_records(s, nullptr), "STR_IN node %d: the literal is not a [count][length][bytes]... record list", i);
      break;
    case SB_OP_STR_LIKE:
      SB_REQUIRE(nd.arg2 >= 1 && nd.arg2 <= 0xFFFF, "STR_LIKE node %d: escape character %d is not a code point in 1..0xFFFF", i, nd.arg2);
      like_segments(s, nd.arg2, i);
      break;
    case SB_OP_STR_OCTET_LENGTH: case SB_OP_STR_CHAR_LENGTH:
      SB_REQUIRE(nd.lit.i == 0 && nd.arg2 == 0, "%s node %d takes no literal", nd.op == SB_OP_STR_OCTET_LENGTH ? "STR_OCTET_LENGTH" : "STR_CHAR_LENGTH", i);
      break;
    default: SB_REQUIRE(nd.arg2 == 0, "string test node %d: arg2 %d must be 0", i, nd.arg2);
  }
  return want;
}

StrTests strpred_compile(const sb_expr &e) {
  StrTests t;
  t.ref.assign(e.n, 0);
  auto put_bytes = [&](const uint8_t *p, uint32_t len) {   // word-aligned; returns the byte offset
    const size_t at = t.words.size();
    t.words.resize(at + (len + 3) / 4, 0u);
    if (len) memcpy(t.words.data() + at, p, len);
    return (uint32_t)(at * 4);
  };
  for (int i = 0; i < e.n; i++) {
    const sb_expr_node &nd = e.nodes[i];
    if (!strpred_is_leaf(nd.op) || strpred_is_length(nd.op)) continue;
    const Slice s = slice_of(e, nd);
    if (nd.op == SB_OP_STR_IN) {
      std::vector<Slice> lits;
      in_records(s, &lits);
      std::sort(lits.begin(), lits.end(), binary_less);
      lits.erase(std::unique(lits.begin(), lits.end(), [](const Slice &a, const Slice &b) { return !binary_less(a, b) && !binary_less(b, a); }),
                 lits.end());
      std::vector<uint32_t> d{(uint32_t)lits.size()};
      for (const Slice &l : lits) {
        d.push_back(put_bytes(l.p, l.len));
        d.push_back(l.len);
      }
      t.ref[i] = (uint32_t)t.words.size();
      t.words.insert(t.words.end(), d.begin(), d.end());
    } else if (nd.op == SB_OP_STR_LIKE) {
      const auto segs = like_segments(s, nd.arg2, i);
      std::vector<uint32_t> d{(uint32_t)segs.size(), segs.size() > 1 ? 1u : 0u};
      for (const auto &u : segs) {
        d.push_back(put_bytes((const uint8_t *)u.data(), (uint32_t)(u.size() * 2)));
        d.push_back((uint32_t)u.size());
      }
      t.ref[i] = (uint32_t)t.words.size();
      t.words.insert(t.words.end(), d.begin(), d.end());
    } else {
      t.ref[i] = (uint32_t)t.words.size();
      t.words.push_back(s.len);
      put_bytes(s.p, s.len);
    }
    SB_REQUIRE(t.words.size() < (1u << 29), "string literals of the expression exceed 2 GB");
  }
  return t;
}

StrBlob::StrBlob(const StrTests &t, cudaStream_t st) : dev((int64_t)t.words.size() * 4, st) {
  // pageable source: the copy has read the host words when the call returns
  if (!t.words.empty()) SB_CUDA(cudaMemcpyAsync(dev.ptr, t.words.data(), t.words.size() * 4, cudaMemcpyHostToDevice, st));
}

}  // namespace sb
