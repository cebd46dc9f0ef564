// join.cu -- equi-joins on the GPU: hash build / probe replacing BroadcastHashJoinExec, ShuffledHashJoinExec
// and SortMergeJoinExec.
//
// Reference path replaced (citations relative to the reference tree, SQLX = sql/core/src/main/scala/org/
// apache/spark/sql/execution):
//   HashedRelation.apply SQLX/joins/HashedRelation.scala:136-168 (LongToUnsafeRowMap :536 for a single long
//   key, UnsafeHashedRelation :209 over BytesToBytesMap otherwise; duplicate keys chain),
//   key packing HashJoin.rewriteKeyExpr SQLX/joins/HashJoin.scala:891-912 (integral keys totalling <= 8 bytes
//   are shifted into one long -- the same packing is used here),
//   probe loops HashJoin.innerJoin :184, outerJoin :215, semiJoin :275, antiJoin :334;
//   a row with any NULL key never matches (HashJoin.scala:160-172);
//   SortMergeJoinScanner SQLX/joins/SortMergeJoinExec.scala:1213-1360 yields the same multiset.
//
// GPU design (random-access bound; HBM for the probe stream, L2/HBM for the table):
//   build : open addressing, capacity = 2^k >= 2 x build rows, linear probing; a build row claims the first
//           free slot of its probe sequence with one 32-bit atomicCAS on the slot's row id (0xFFFFFFFF = free)
//           and then stores its packed 64-bit key -- duplicates simply occupy several slots; no sentinel key.
//           A slot is 16 bytes {key, row id}, so a probe step is ONE 128-bit load (one 32-byte sector).
//   probe : pass 1 counts matches per streamed row (and remembers the first match), exclusive scan,
//           pass 2 writes (probe row, build row) pairs in streamed-row order; rows with <= 1 match do not walk
//           the table twice.  Output columns are gathered once from both sides.
#include <memory>
#include "common.cuh"
#include "expr.cuh"
#include "simple_pred.cuh"
#include "primitives.cuh"
#include "rtc.cuh"
#include "strings.cuh"

struct sb_hash_table {
  sb_table *build = nullptr;        // retained build-side batch (payload gathered at probe time)
  struct Slot { uint64_t key; uint32_t row; uint32_t pad; };   // 16 bytes: one sector-aligned load per probe step
  Slot *slots = nullptr;            // [cap]; row == 0xFFFFFFFF means free
  int64_t cap = 0;
  int32_t nkeys = 0;
  int32_t key_col[4];                 // build-side column index of every key
  int32_t key_type[4];
  int32_t key_bits[4];
  int32_t key_shift[4];
  int32_t *null_key_flag = nullptr;   // device: set when a build row had a NULL key (null-aware anti join)
  // prefilter in front of the table, one of:
  //   exact  -- a bitmap over [fmin, fmin + frange) of the packed key: bit (key - fmin) set <=> the key is in the relation.  Chosen
  //             when the key range is dense enough (<= 64 bits per key); the analogue of LongToUnsafeRowMap's dense mode
  //             (SQLX/joins/HashedRelation.scala:535-1010, optimize()), used as a filter in front of the open-addressing table.
  //             A streamed side clustered on the key (lineitem by l_orderkey) walks it sequentially.
  //   Bloom  -- blocked: one 32-bit word per key hash, 3 bits set; at most 32 MB so that it stays resident in H100's 50 MB L2
  uint32_t *bloom = nullptr;
  uint64_t bloom_mask = 0;            // Bloom: words - 1 (power of two)
  int exact = 0;
  uint64_t fmin = 0, frange = 0;
  // exact relations know whether their keys are unique (a bit that is already set when a key arrives = a duplicate).  Unique keys
  // turn the probe into one lookup per candidate (no count / scan / fill); a dense key range (<= 8 slots of range per key) also
  // replaces the open-addressing table by a direct-address one, row_of[key - fmin] -- LongToUnsafeRowMap's dense mode proper.
  int unique = 0;
  uint32_t *row_of = nullptr;         // dense mode: [frange], FREE_SLOT = no such key; slots is NULL then
  // sorted mode: the build rows arrive with strictly ascending keys (the output of a join over a key-ordered scan, a primary-key
  // scan ...), so the row of a key is its RANK among the set bits of the bitmap: rank[w] = set bits before word w.  No slots.
  uint32_t *rank = nullptr;
  int64_t nkeys_in = 0;               // build rows that entered the relation (filter TRUE, keys not NULL)
  // string key columns join as int32 codes in the BUILD side's dictionaries (csrc/strings.cu): has_dict[i] says key i is one
  bool has_dict[4] = {false, false, false, false};
  sb::Column dict[4];
  // wide keys (> 64 bits): the slots hold a hash; the key columns of the build side stay reachable for the verification
  int wide = 0;
  sb_table *key_table = nullptr;      // retained table the build key columns live in (the build table or its encoded view)
  int32_t key_table_col[4] = {0, 0, 0, 0};
  cudaStream_t st = nullptr;
  cudaEvent_t ready = nullptr;        // recorded on `st` when the build's device work has been enqueued: probes on OTHER streams wait for it
};

namespace sb {

constexpr int JOIN_THREADS = 256;
constexpr int JOIN_MAX_KEYS = 4;
constexpr uint32_t FREE_SLOT = 0xFFFFFFFFu;

struct JoinKeys {
  int n;
  const void *data[JOIN_MAX_KEYS];
  const uint8_t *valid[JOIN_MAX_KEYS];
  int32_t type[JOIN_MAX_KEYS];
  int32_t bits[JOIN_MAX_KEYS];
  int32_t shift[JOIN_MAX_KEYS];
  int32_t wide;   // the key columns need more than 64 bits: join_key yields a 64-bit HASH of them and matches are verified
                  // column by column against the build row (the general UnsafeHashedRelation case of HashedRelation.scala:136)
};

__device__ __forceinline__ uint64_t join_mix(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// normalised value of key column i of a row (-0.0 == 0.0, one NaN, like grouping keys), zero-extended to its width
__device__ __forceinline__ uint64_t join_key_part(const JoinKeys &k, int i, int64_t row) {
  if (k.type[i] == SB_FLOAT64) {
    double d = ((const double *)k.data[i])[row];
    return d == 0.0 ? 0ull : (uint64_t)double_bits_canonical(d);
  }
  if (k.type[i] == SB_FLOAT32) {
    float f = ((const float *)k.data[i])[row];
    return f == 0.0f ? 0u : (uint32_t)float_bits_canonical(f);
  }
  uint64_t v = (uint64_t)load_i64(k.data[i], k.type[i], row);
  if (k.bits[i] < 64) v &= (1ull << k.bits[i]) - 1;
  return v;
}
// packed key of a row (wide keys: a hash of the parts); false when any key column is NULL (such a row never matches)
__device__ __forceinline__ bool join_key(const JoinKeys &k, int64_t row, uint64_t &out) {
  uint64_t w = 0;
#pragma unroll
  for (int i = 0; i < JOIN_MAX_KEYS; i++) {
    if (i >= k.n) break;
    if (!bit_valid(k.valid[i], row)) return false;
    const uint64_t v = join_key_part(k, i, row);
    if (k.wide) w = join_mix(w ^ v) + (uint64_t)i;
    else w |= v << k.shift[i];
  }
  out = w;
  return true;
}
// wide keys: do the key columns of streamed row `row` equal those of build row `brow`?  (narrow keys: the packed words did)
__device__ __forceinline__ bool join_key_verify(const JoinKeys &k, int64_t row, const JoinKeys &bk, int64_t brow) {
  if (!k.wide) return true;
#pragma unroll
  for (int i = 0; i < JOIN_MAX_KEYS; i++) {
    if (i >= k.n) break;
    if (join_key_part(k, i, row) != join_key_part(bk, i, brow)) return false;
  }
  return true;
}

// Blocked Bloom filter in front of the table.  A selective join (Q3: one streamed row in ten has a partner) would otherwise
// pay a random 32-byte HBM sector per streamed row just to learn "no": the filter is at most 32 MB, i.e. L2-resident, and
// answers that for ~99.9 % of the rows without a partner with one L2 access.
__device__ __forceinline__ uint32_t bloom_bits(uint64_t h) {
  return (1u << (h >> 59)) | (1u << ((h >> 54) & 31)) | (1u << ((h >> 49) & 31));
}
__device__ __forceinline__ uint64_t bloom_word(uint64_t h, uint64_t mask) { return (h >> 20) & mask; }

struct KeyFilter {
  const uint32_t *words;
  uint64_t mask, fmin, frange;
  int exact;
  const uint32_t *row_of;   // dense direct-address table (implies exact, unique keys)
  const uint32_t *rank;     // sorted mode: set bits before every bitmap word (implies exact, unique keys)
};
// build row of a key the exact prefilter has confirmed, for the relations that keep no slot table
__device__ __forceinline__ uint32_t direct_row(const KeyFilter &f, uint64_t key) {
  const uint64_t d = key - f.fmin;
  if (f.row_of) return __ldg(&f.row_of[d]);
  return __ldg(&f.rank[d >> 5]) + (uint32_t)__popc(__ldg(&f.words[d >> 5]) & ((1u << (d & 31)) - 1u));
}
__device__ __forceinline__ bool filter_test(const KeyFilter &f, uint64_t key) {
  if (!f.words) return true;
  if (f.exact) {
    const uint64_t d = key - f.fmin;
    return d < f.frange && ((__ldg(&f.words[d >> 5]) >> (d & 31)) & 1u);
  }
  const uint64_t hh = join_mix(key);
  const uint32_t bb = bloom_bits(hh);
  return (__ldg(&f.words[bloom_word(hh, f.mask)]) & bb) == bb;
}

// Runtime filters (the reference's InjectRuntimeFilter, sql/catalyst/.../optimizer/InjectRuntimeFilter.scala:47-100: a
// BloomFilterMightContain FilterExec on the application side of a join, built from the creation side's join keys): here the filter
// IS the prefilter of a single-key relation built on the creation side (exact bitmap or Bloom).  Long streamed sides: the join's own
// candidate pass runs first and the filter is applied to the candidate LIST (runtime_filter_rows_kernel + a compaction) -- the extra
// column is read only for the rows the join's prefilter let through.  Testing it inside the candidate pass was measured and dropped:
// the straight-line test costs every row ~40 instructions (it doubled the time of Q5's lineitem pass).  Short streamed
// sides: a byte mask like a fused FilterExec's (runtime_filter_mask_kernel).

typedef sb_hash_table::Slot JoinSlot;
__device__ __forceinline__ void load_slot(const JoinSlot *p, uint64_t &key, uint32_t &row) {
  const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(p);
  key = v.x;
  row = (uint32_t)v.y;
}

__global__ void __launch_bounds__(JOIN_THREADS) join_build_kernel(JoinKeys k, int64_t n, JoinSlot *__restrict__ slots, int64_t cap,
                                                                  int32_t *__restrict__ null_key_flag, const uint8_t *__restrict__ row_mask,
                                                                  KeyFilter kf) {
  int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n) return;
  if (row_mask && !row_mask[row]) return;   // fused FilterExec below the build side: the row is not part of the relation
  uint64_t key;
  if (!join_key(k, row, key)) {
    *null_key_flag = 1;   // HashedRelation keeps no NULL keys; the null-aware anti join needs to know there was one
    return;
  }
  uint64_t mask = (uint64_t)cap - 1;
  const uint64_t hh = join_mix(key);
  uint64_t h = hh & mask;
  uint32_t *fw = const_cast<uint32_t *>(kf.words);
  if (kf.exact) {
    const uint64_t d = key - kf.fmin;
    const uint32_t bit = 1u << (d & 31);
    if (atomicOr(&fw[d >> 5], bit) & bit) null_key_flag[1] = 1;   // the key was there already: the relation is not unique
    if (kf.row_of) {   // dense mode: the direct-address table is the relation (a duplicate voids it; the host rebuilds)
      const_cast<uint32_t *>(kf.row_of)[d] = (uint32_t)row;
      return;
    }
    if (!slots) return;   // sorted mode: the bitmap (+ its rank prefix) is the relation
  } else if (fw) atomicOr(&fw[bloom_word(hh, kf.mask)], bloom_bits(hh));
  for (;;) {
    if (slots[h].row == FREE_SLOT && atomicCAS(&slots[h].row, FREE_SLOT, (uint32_t)row) == FREE_SLOT) {
      slots[h].key = key;
      return;
    }
    h = (h + 1) & mask;
  }
}

// pass 1: matches per streamed row (join-type adjusted) + first matching build row
__global__ void __launch_bounds__(JOIN_THREADS) join_count_kernel(JoinKeys k, int64_t n, const JoinSlot *__restrict__ slots, int64_t cap,
                                                                  int join_type, int null_aware, int32_t *__restrict__ counts, uint32_t *__restrict__ first,
                                                                  int32_t *__restrict__ block_counts, uint8_t *__restrict__ matched,
                                                                  const uint8_t *__restrict__ row_mask, KeyFilter kf,
                                                                  const int64_t *__restrict__ rows, JoinKeys bk) {
  __shared__ int32_t wsum[JOIN_THREADS / 32];
  // `rows` (optional): the candidate list of join_candidate_kernel -- item i stands for streamed row rows[i]; counts / first are
  // indexed by item
  const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = rows && item < n ? rows[item] : item;
  const bool in_range = item < n && (!row_mask || row_mask[row]);   // fused FilterExec below the streamed side
  uint64_t key;
  int32_t matches = 0;
  uint32_t f = FREE_SLOT;
  bool null_key = false;
  if (in_range) {
    if (join_key(k, row, key)) {
      uint64_t mask = (uint64_t)cap - 1;
      const uint64_t hh = join_mix(key);
      uint64_t h = hh & mask;
      if (filter_test(kf, key)) {
        if (kf.row_of || kf.rank) {   // dense / sorted, unique: the prefilter said the key exists
          f = direct_row(kf, key);
          matches = 1;
          if (matched) matched[f] = 1;
        } else
        for (;;) {
          uint64_t sk;
          uint32_t r;
          load_slot(&slots[h], sk, r);
          if (r == FREE_SLOT) break;
          if (sk == key && join_key_verify(k, row, bk, r)) {
            if (matches == 0) f = r;
            matches++;
            if (matched) matched[r] = 1;   // build rows that found a partner (build-side-preserving outer joins)
          }
          h = (h + 1) & mask;
        }
      }
    } else null_key = true;
  }
  int32_t c;
  switch (join_type) {
    case SB_JOIN_INNER: c = matches; break;
    case SB_JOIN_LEFT_OUTER: c = matches > 0 ? matches : 1; break;
    case SB_JOIN_LEFT_SEMI: c = matches > 0 ? 1 : 0; break;
    case SB_JOIN_EXISTENCE: c = 1; break;      // every streamed row, `first` says whether it has a partner
    default: c = matches > 0 || (null_aware && null_key) ? 0 : 1; break;   // anti (null-aware: a NULL key is neither in nor not in)
  }
  if (!in_range) c = 0;
  if (item < n) {
    first[item] = f;
    counts[item] = c;
  }
  // output rows of this block: the scan that turns counts into offsets runs over blocks, not rows (join_fill_kernel redoes
  // the in-block prefix in shared memory), which saves an 8-byte offset per streamed row and two passes over them
  int32_t t = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t b = 0;
#pragma unroll
    for (int w = 0; w < JOIN_THREADS / 32; w++) b += wsum[w];
    block_counts[blockIdx.x] = b;
  }
}

// pass 2: (probe row, build row) pairs at the scanned offsets
__global__ void __launch_bounds__(JOIN_THREADS) join_fill_kernel(JoinKeys k, int64_t n, const JoinSlot *__restrict__ slots, int64_t cap,
                                                                 int join_type, const int32_t *__restrict__ counts,
                                                                 const int64_t *__restrict__ block_offsets, const uint32_t *__restrict__ first,
                                                                 int64_t *__restrict__ out_probe, int64_t *__restrict__ out_build,
                                                                 const int64_t *__restrict__ rows, JoinKeys bk) {
  __shared__ int32_t wsum[JOIN_THREADS / 32];
  const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = rows && item < n ? rows[item] : item;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int32_t c = item < n ? counts[item] : 0;
  int32_t x = c;   // inclusive prefix inside the warp
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) wsum[warp] = x;
  __syncthreads();
  int32_t woff = 0;
  for (int w = 0; w < warp; w++) woff += wsum[w];
  if (c == 0) return;
  int64_t o = block_offsets[blockIdx.x] + woff + (x - c);
  uint32_t f = first[item];
  if (c == 1 || join_type == SB_JOIN_LEFT_SEMI || join_type == SB_JOIN_LEFT_ANTI) {
    out_probe[o] = row;
    if (out_build) out_build[o] = (f == FREE_SLOT || join_type >= SB_JOIN_LEFT_SEMI) ? -1 : (int64_t)f;
    return;
  }
  uint64_t key;
  join_key(k, row, key);
  uint64_t mask = (uint64_t)cap - 1;
  uint64_t h = join_mix(key) & mask;
  for (;;) {
    uint64_t sk;
    uint32_t r;
    load_slot(&slots[h], sk, r);
    if (r == FREE_SLOT) break;
    if (sk == key && join_key_verify(k, row, bk, r)) {
      out_probe[o] = row;
      out_build[o] = r;
      o++;
    }
    h = (h + 1) & mask;
  }
}

// Selective joins over a long streamed side (Q3: 600 M lineitem rows, one in twenty survives filter + prefilter): ONE pass over
// (pushed-down filter, key, prefilter word) marks the rows that can produce output at all; only those -- as a compacted row list --
// go through the count / fill passes with their per-row bookkeeping.  A thread owns 16 consecutive rows (16-byte loads), writes
// their verdicts as one 16-bit word and the block leaves its candidate count for the scan, so the list is produced by one more
// pass over 1 bit per row.  mode (CandMode): inner / semi joins drop NULL-key and prefilter-negative rows here; outer / anti joins keep
// every row the filter keeps (those rows are output even without a partner).
// (Tried and dropped: a lane-strided layout -- a warp reads 32 consecutive rows per load, verdicts leave as ballot words.  Every
// load was perfectly coalesced, but with the general key / predicate code inlined per row the loads sat behind per-row branches
// and no longer overlapped: Q3's 600 M-row pass became several times slower.  The 16-byte loads below are issued back to back.)
constexpr int CAND_ROWS = SP_ROWS;
// which rows the candidate pass keeps, next to the pushed-down filter
enum CandMode {
  CAND_ALL = 0,           // every row (outer joins; anti joins behind a Bloom filter, which cannot prove absence)
  CAND_PRESENT = 1,       // non-NULL key that passes the prefilter (inner, semi)
  CAND_ABSENT = 2,        // exact prefilter only: NULL key or key not in the relation (anti join: these rows ARE the answer)
  CAND_ABSENT_KEYED = 3   // exact prefilter only: non-NULL key not in the relation (null-aware anti join)
};
constexpr int CAND_TILE = JOIN_THREADS * CAND_ROWS;
__global__ void __launch_bounds__(JOIN_THREADS) join_candidate_kernel(JoinKeys k, int64_t n, const __grid_constant__ SimplePred sp,
                                                                      const uint8_t *__restrict__ row_mask, KeyFilter kf, int mode,
                                                                      int fast_key, uint16_t *__restrict__ bits_out,
                                                                      int32_t *__restrict__ block_counts) {
  __shared__ int32_t wsum[JOIN_THREADS / 32];
  const int64_t row0 = ((int64_t)blockIdx.x * JOIN_THREADS + threadIdx.x) * CAND_ROWS;
  uint32_t keep = 0;
  if (row0 < n) {
    keep = row0 + CAND_ROWS <= n ? 0xFFFFu : (1u << (int)(n - row0)) - 1u;
    if (sp.nterms > 0) keep &= simple_pred_eval16(sp, row0, n);
    if (row_mask) {
      uint32_t mbits = 0;
      if (row0 + CAND_ROWS <= n) {   // scratch masks are 16-byte aligned and row0 is a multiple of 16
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(row_mask + row0));
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < CAND_ROWS; j++) mbits |= (((w[j >> 2] >> (8 * (j & 3))) & 0xFFu) ? 1u : 0u) << j;
      } else {
        for (int j = 0; row0 + j < n; j++) mbits |= (row_mask[row0 + j] ? 1u : 0u) << j;
      }
      keep &= mbits;
    }
    if (mode != CAND_ALL) {
      uint64_t key[CAND_ROWS];
      uint32_t has = 0xFFFFu;
      if (fast_key) {   // one NULL-free integer key column: the 16 keys arrive as 16-byte loads whatever `keep` says
        int64_t x[CAND_ROWS];
        switch (k.type[0]) {
          case SB_INT8: sp_load16<int8_t>(k.data[0], row0, n, x); break;
          case SB_INT16: sp_load16<int16_t>(k.data[0], row0, n, x); break;
          case SB_INT32: case SB_DATE32: sp_load16<int32_t>(k.data[0], row0, n, x); break;
          default: sp_load16<int64_t>(k.data[0], row0, n, x); break;
        }
        const uint64_t km = k.bits[0] < 64 ? (1ull << k.bits[0]) - 1 : ~0ull;
#pragma unroll
        for (int j = 0; j < CAND_ROWS; j++) key[j] = (uint64_t)x[j] & km;
      } else {
        has = 0;
#pragma unroll
        for (int j = 0; j < CAND_ROWS; j++) {
          key[j] = 0;
          if (((keep >> j) & 1u) && join_key(k, row0 + j, key[j])) has |= 1u << j;
        }
      }
      uint32_t present = has;   // rows whose key is (or, with a Bloom filter, may be) in the relation
      if (kf.words) {
        present = 0;
#pragma unroll
        for (int j = 0; j < CAND_ROWS; j++)
          if (((keep & has) >> j) & 1u) present |= (filter_test(kf, key[j]) ? 1u : 0u) << j;
      }
      keep &= mode == CAND_PRESENT ? present : mode == CAND_ABSENT ? ~present : (has & ~present);
    }
    bits_out[row0 / CAND_ROWS] = (uint16_t)keep;
  }
  int32_t t = __reduce_add_sync(0xffffffffu, __popc(keep));
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t b = 0;
#pragma unroll
    for (int w = 0; w < JOIN_THREADS / 32; w++) b += wsum[w];
    block_counts[blockIdx.x] = b;
  }
}

// Variant (sb_config_set("join_cand", 1)): lane-strided.  A warp owns 512 consecutive rows of the block's 4096 and visits them 32 at
// a time -- lane l reads row base + l, so every column load is one coalesced warp-wide access -- 8 such groups per step, and inside
// a step every stage issues ALL its loads before the first use (keys, then predicate terms one by one, then prefilter words), so
// they overlap.  The verdicts of 32 rows are one ballot word = two of the 16-bit words candidate_rows_kernel reads (little endian),
// so the bits buffer, the block counts and the second kernel are shared with the variant above.
// KW: 0 = general keys (join_key per row), 4 / 8 = ONE NULL-free integer key column of that width.
// join_key for R rows at once, column by column: the R loads of a column are issued together and its type switch is outside the
// row loop (the per-row join_key puts every load behind a branch).  has[j]: no key column of row j is NULL.
template <int R>
__device__ __forceinline__ void join_key_rows(const JoinKeys &k, const int64_t (&rr)[R], uint64_t (&key)[R], bool (&has)[R]) {
#pragma unroll
  for (int j = 0; j < R; j++) {
    key[j] = 0;
    has[j] = true;
  }
#pragma unroll
  for (int i = 0; i < JOIN_MAX_KEYS; i++) {   // unrolled: the per-column fields of the kernel parameter are indexed statically
    if (i >= k.n) break;
    if (k.valid[i]) {
      uint8_t vb[R];
#pragma unroll
      for (int j = 0; j < R; j++) vb[j] = k.valid[i][rr[j] >> 3];
#pragma unroll
      for (int j = 0; j < R; j++) has[j] = has[j] && ((vb[j] >> (rr[j] & 7)) & 1);
    }
    uint64_t v[R];
    switch (k.type[i]) {
      case SB_FLOAT64:
#pragma unroll
        for (int j = 0; j < R; j++) {
          const double d = ((const double *)k.data[i])[rr[j]];
          v[j] = d == 0.0 ? 0ull : (uint64_t)double_bits_canonical(d);
        }
        break;
      case SB_FLOAT32:
#pragma unroll
        for (int j = 0; j < R; j++) {
          const float f = ((const float *)k.data[i])[rr[j]];
          v[j] = f == 0.0f ? 0u : (uint32_t)float_bits_canonical(f);
        }
        break;
      case SB_INT64: case SB_TIMESTAMP: case SB_DECIMAL64:
#pragma unroll
        for (int j = 0; j < R; j++) v[j] = ((const uint64_t *)k.data[i])[rr[j]];
        break;
      case SB_INT32: case SB_DATE32:
#pragma unroll
        for (int j = 0; j < R; j++) v[j] = ((const uint32_t *)k.data[i])[rr[j]];
        break;
      default: {
        const uint64_t m = k.bits[i] < 64 ? (1ull << k.bits[i]) - 1 : ~0ull;
#pragma unroll
        for (int j = 0; j < R; j++) v[j] = (uint64_t)load_i64(k.data[i], k.type[i], rr[j]) & m;
      }
    }
    if (k.wide) {
#pragma unroll
      for (int j = 0; j < R; j++) key[j] = join_mix(key[j] ^ v[j]) + (uint64_t)i;
    } else {
      const int sh = k.shift[i];
#pragma unroll
      for (int j = 0; j < R; j++) key[j] |= v[j] << sh;
    }
  }
}

template <int KW, bool FULL, int CAND_STEP>
__device__ __forceinline__ uint32_t candidate_step(const JoinKeys &k, int64_t n, const SimplePred &sp, const uint8_t *__restrict__ row_mask,
                                                   const KeyFilter &kf, int mode, int64_t g0, int lane, uint32_t (&words)[CAND_STEP]) {
  // rows of this lane: g0 + lane + 32 j.  FULL: the whole step lies below n, so nothing is clamped and the column pointers are
  // advanced once (the loads take constant offsets)
  const int64_t r0 = g0 + lane;
  bool keep[CAND_STEP], has[CAND_STEP];
  uint64_t key[CAND_STEP];
  int64_t rr[CAND_STEP];
#pragma unroll
  for (int j = 0; j < CAND_STEP; j++) {
    const int64_t r = r0 + (int64_t)j * 32;
    keep[j] = FULL || r < n;
    rr[j] = FULL || r < n ? r : n - 1;
    has[j] = true;
  }
  if (mode != CAND_ALL) {   // the key loads do not wait for the filter's verdict
    if (KW == 8) {
      const uint64_t *p = (const uint64_t *)k.data[0] + (FULL ? r0 : 0);
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) key[j] = FULL ? p[j * 32] : p[rr[j]];
    } else if (KW == 4) {
      const uint32_t *p = (const uint32_t *)k.data[0] + (FULL ? r0 : 0);
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) key[j] = (uint64_t)(FULL ? p[j * 32] : p[rr[j]]);
    } else {
      join_key_rows<CAND_STEP>(k, rr, key, has);
    }
  }
  if (sp.nterms > 0) simple_pred_rows<CAND_STEP, FULL>(sp, r0, 32, n, keep);
  if (row_mask) {
    uint8_t m[CAND_STEP];
#pragma unroll
    for (int j = 0; j < CAND_STEP; j++) m[j] = row_mask[rr[j]];
#pragma unroll
    for (int j = 0; j < CAND_STEP; j++) keep[j] = keep[j] && m[j] != 0;
  }
  if (mode != CAND_ALL) {
    bool present[CAND_STEP];
#pragma unroll
    for (int j = 0; j < CAND_STEP; j++) present[j] = has[j] && keep[j];
    if (kf.words && kf.exact) {   // frange <= 2^31: inside the range the offset is a 32-bit number
      uint32_t w[CAND_STEP], d[CAND_STEP];
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) {
        const uint64_t d64 = key[j] - kf.fmin;
        present[j] = present[j] && d64 < kf.frange;
        d[j] = (uint32_t)d64;
        w[j] = present[j] ? __ldg(&kf.words[d[j] >> 5]) : 0u;
      }
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) present[j] = present[j] && ((w[j] >> (d[j] & 31)) & 1u);
    } else if (kf.words) {
      uint32_t w[CAND_STEP], bb[CAND_STEP];
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) {
        const uint64_t hh = join_mix(key[j]);
        bb[j] = bloom_bits(hh);
        w[j] = present[j] ? __ldg(&kf.words[bloom_word(hh, kf.mask)]) : 0u;
      }
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) present[j] = present[j] && (w[j] & bb[j]) == bb[j];
    }
    if (mode == CAND_PRESENT) {
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) keep[j] = present[j];          // present implies keep
    } else if (mode == CAND_ABSENT) {
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) keep[j] = keep[j] && !present[j];
    } else {
#pragma unroll
      for (int j = 0; j < CAND_STEP; j++) keep[j] = keep[j] && has[j] && !present[j];
    }
  }
  uint32_t count = 0;
#pragma unroll
  for (int j = 0; j < CAND_STEP; j++) {
    words[j] = __ballot_sync(0xffffffffu, keep[j]);
    count += __popc(words[j]);
  }
  return count;
}
// the ragged last step of the input: kept out of line so that its clamping code costs the full steps no registers
template <int KW, int CAND_STEP>
__device__ __noinline__ uint32_t candidate_step_tail(const JoinKeys &k, int64_t n, const SimplePred &sp, const uint8_t *__restrict__ row_mask,
                                                     const KeyFilter &kf, int mode, int64_t g0, int lane, uint32_t (&words)[CAND_STEP]) {
  return candidate_step<KW, false, CAND_STEP>(k, n, sp, row_mask, kf, mode, g0, lane, words);
}
template <int KW, int CAND_STEP, int MINB>
__global__ void __launch_bounds__(JOIN_THREADS, MINB) join_candidate_strided_kernel(JoinKeys k, int64_t n, const __grid_constant__ SimplePred sp,
                                                                              const uint8_t *__restrict__ row_mask, KeyFilter kf, int mode,
                                                                              uint32_t *__restrict__ bits_out, int32_t *__restrict__ block_counts) {
  __shared__ int32_t wsum[JOIN_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int WARP_ROWS = CAND_TILE / (JOIN_THREADS / 32);
  const int64_t wbase = (int64_t)blockIdx.x * CAND_TILE + (int64_t)warp * WARP_ROWS;
  uint32_t mine = 0;
#pragma unroll 1
  for (int c = 0; c < WARP_ROWS / 32; c += CAND_STEP) {
    const int64_t g0 = wbase + (int64_t)c * 32;
    if (g0 >= n) break;
    uint32_t words[CAND_STEP];
    const uint32_t cnt = g0 + CAND_STEP * 32 <= n ? candidate_step<KW, true, CAND_STEP>(k, n, sp, row_mask, kf, mode, g0, lane, words)
                                                   : candidate_step_tail<KW, CAND_STEP>(k, n, sp, row_mask, kf, mode, g0, lane, words);
    mine += cnt;   // the same on every lane
#pragma unroll
    for (int j = 0; j < CAND_STEP; j++)
      if (lane == j && g0 + (int64_t)j * 32 < n) bits_out[(g0 >> 5) + j] = words[j];
  }
  if (lane == 0) wsum[warp] = (int32_t)mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t b = 0;
#pragma unroll
    for (int w = 0; w < JOIN_THREADS / 32; w++) b += wsum[w];
    block_counts[blockIdx.x] = b;
  }
}

// the candidate list in row order: same tiling as join_candidate_kernel, block_offsets = exclusive scan of its block counts
__global__ void __launch_bounds__(JOIN_THREADS) candidate_rows_kernel(const uint16_t *__restrict__ bits, int64_t nwords,
                                                                      const int64_t *__restrict__ block_offsets, int64_t *__restrict__ rows) {
  __shared__ int32_t wsum[JOIN_THREADS / 32];
  const int64_t t = (int64_t)blockIdx.x * JOIN_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t b = t < nwords ? bits[t] : 0u;
  const int32_t c = __popc(b);
  int32_t x = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) wsum[warp] = x;
  __syncthreads();
  int32_t woff = 0;
  for (int w = 0; w < warp; w++) woff += wsum[w];
  int64_t o = block_offsets[blockIdx.x] + woff + (x - c);
  const int64_t row0 = t * CAND_ROWS;
  while (b) {
    const int j = __ffs(b) - 1;
    b &= b - 1;
    rows[o++] = row0 + j;
  }
}

// Relations with unique keys behind an exact prefilter: one lookup per candidate gives its partner -- no count / scan / fill.
// outer: candidates without a partner (NULL key or key not in the relation) get -1.
__global__ void __launch_bounds__(JOIN_THREADS) join_lookup_kernel(JoinKeys k, const int64_t *__restrict__ rows, int64_t nitems,
                                                                   const JoinSlot *__restrict__ slots, int64_t cap, KeyFilter kf, int outer,
                                                                   int64_t *__restrict__ out_build) {
  const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= nitems) return;
  const int64_t row = rows[item];
  uint64_t key;
  int64_t found = -1;
  if (join_key(k, row, key) && (!outer || filter_test(kf, key))) {   // not outer: the candidate pass has done the test
    if (kf.row_of || kf.rank) found = (int64_t)direct_row(kf, key);
    else {
      const uint64_t mask = (uint64_t)cap - 1;
      uint64_t h = join_mix(key) & mask;
      for (;;) {
        uint64_t sk;
        uint32_t r;
        load_slot(&slots[h], sk, r);
        if (r == FREE_SLOT) break;
        if (sk == key) {
          found = (int64_t)r;
          break;
        }
        h = (h + 1) & mask;
      }
    }
  }
  out_build[item] = found;
}

// what the relation will hold: packed-key range and row count of the build rows that pass the filter with non-NULL keys
// stats[3] != 0: the rows do not arrive with strictly ascending keys (checked only without a filter: every row is in the relation)
__global__ void __launch_bounds__(JOIN_THREADS) build_stats_kernel(JoinKeys k, int64_t n, const uint8_t *__restrict__ row_mask,
                                                                   long long *__restrict__ stats) {
  long long lo = 0x7FFFFFFFFFFFFFFFll, hi = -0x7FFFFFFFFFFFFFFFll - 1, cnt = 0;
  bool unsorted = false;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    if (row_mask && !row_mask[row]) continue;
    uint64_t key;
    if (!join_key(k, row, key)) {
      unsorted = true;
      continue;
    }
    if (!row_mask && row > 0) {
      uint64_t prev;
      if (!join_key(k, row - 1, prev) || (long long)prev >= (long long)key) unsorted = true;
    }
    const long long v = (long long)key;
    lo = v < lo ? v : lo;
    hi = v > hi ? v : hi;
    cnt++;
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    const long long l2 = __shfl_xor_sync(0xffffffffu, lo, d), h2 = __shfl_xor_sync(0xffffffffu, hi, d);
    lo = l2 < lo ? l2 : lo;
    hi = h2 > hi ? h2 : hi;
    cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  }
  if ((threadIdx.x & 31) == 0 && cnt > 0) {
    atomicMin(&stats[0], lo);
    atomicMax(&stats[1], hi);
    atomicAdd((unsigned long long *)&stats[2], (unsigned long long)cnt);
  }
  if (__any_sync(0xffffffffu, unsorted) && (threadIdx.x & 31) == 0) stats[3] = 1;
}
__global__ void word_popc_kernel(const uint32_t *__restrict__ words, int64_t n, int32_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __popc(words[i]);
}

// runtime filter outside the candidate pass (short streamed sides, nullable or odd-typed columns): a byte mask like a fused FilterExec's
__global__ void __launch_bounds__(JOIN_THREADS) runtime_filter_mask_kernel(JoinKeys col, int64_t n, KeyFilter f, uint8_t *__restrict__ mask, int have_mask) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n) return;
  if (have_mask && !mask[row]) return;
  uint64_t key;
  mask[row] = join_key(col, row, key) && filter_test(f, key) ? 1 : 0;   // might_contain(NULL) is NULL: the row is dropped
}

__global__ void __launch_bounds__(JOIN_THREADS) runtime_filter_rows_kernel(JoinKeys col, const int64_t *__restrict__ rows, int64_t nitems, KeyFilter f,
                                                                           uint8_t *__restrict__ flags, int have_flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nitems) return;
  if (have_flags && !flags[i]) return;
  uint64_t key;
  flags[i] = join_key(col, rows[i], key) && filter_test(f, key) ? 1 : 0;
}
__global__ void __launch_bounds__(JOIN_THREADS) take_rows_kernel(const int64_t *__restrict__ rows, const int64_t *__restrict__ idx, int64_t m, int64_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) out[i] = rows[idx[i]];
}

static KeyFilter key_filter_of(const sb_hash_table *ht) {
  KeyFilter f;
  f.words = ht->bloom;
  f.mask = ht->bloom_mask;
  f.fmin = ht->fmin;
  f.frange = ht->frange;
  f.exact = ht->exact;
  f.row_of = ht->row_of;
  f.rank = ht->rank;
  return f;
}

static JoinKeys make_join_keys(const sb_table *t, const int32_t *key_cols, int32_t nkeys, const sb_hash_table *ht) {
  SB_REQUIRE(nkeys >= 1 && nkeys <= JOIN_MAX_KEYS, "joins support 1..%d key columns (got %d)", JOIN_MAX_KEYS, nkeys);
  JoinKeys k;
  k.n = nkeys;
  int pos = 0;
  for (int i = 0; i < nkeys; i++) {
    SB_REQUIRE(key_cols[i] >= 0 && key_cols[i] < (int)t->cols.size(), "join key column %d out of range", key_cols[i]);
    const Column &c = t->cols[key_cols[i]];
    SB_REQUIRE(c.type != SB_STRING, "string join keys reach the kernels as dictionary codes");
    if (c.type == SB_DECIMAL128) fail(SB_ERR_UNSUPPORTED, "decimal(p > 18) join keys are not supported");
    k.data[i] = c.d();
    k.valid[i] = c.v();
    k.type[i] = c.type;
    int bits = type_width(c.type) * 8;
    if (ht) {   // the probe side must pack exactly like the build side
      SB_REQUIRE(ht->key_bits[i] == bits, "join key %d: probe width %d bits differs from build width %d bits (cast first)", i, bits,
                 ht->key_bits[i]);
    }
    k.bits[i] = bits;
    k.shift[i] = pos;
    pos += bits;
  }
  // <= 64 bits: the key columns are packed into one word (HashJoin.rewriteKeyExpr, HashJoin.scala:715-760 -> LongHashedRelation);
  // more: the slots hold a 64-bit hash and every hash match is verified against the build row's key columns (UnsafeHashedRelation)
  k.wide = pos > 64;
  if (ht) SB_REQUIRE((ht->wide != 0) == (k.wide != 0), "join keys: the streamed side packs to %d bits, the relation was built %s", pos, ht->wide ? "wide" : "narrow");
  return k;
}

// key columns of the BUILD side for the verification of wide-key matches (narrow keys: unused, a zeroed struct)
static JoinKeys build_side_keys(const sb_hash_table *ht) {
  JoinKeys bk;
  memset(&bk, 0, sizeof(bk));
  if (!ht->wide) return bk;
  bk.n = ht->nkeys;
  bk.wide = 1;
  for (int i = 0; i < ht->nkeys; i++) {
    const Column &c = ht->key_table->cols[ht->key_table_col[i]];
    bk.data[i] = c.d();
    bk.valid[i] = c.v();
    bk.type[i] = c.type;
    bk.bits[i] = ht->key_bits[i];
    bk.shift[i] = 0;
  }
  return bk;
}

// The table the streamed side's keys are read from: `probe` itself, or a view in which the string key columns hold their codes in
// the relation's dictionaries (a string the build side never saw gets -1: it equals no build code, so outer / anti joins still
// emit the row).
static const sb_table *probe_key_source(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys, cudaStream_t st,
                                        EncodedView &ev) {
  std::vector<int> cols;
  std::vector<const Column *> dicts;
  for (int i = 0; i < nkeys && i < JOIN_MAX_KEYS; i++) {
    SB_REQUIRE(key_cols[i] >= 0 && key_cols[i] < (int)probe->cols.size(), "join key column %d out of range", key_cols[i]);
    const bool is_str = probe->cols[key_cols[i]].type == SB_STRING;
    SB_REQUIRE(is_str == ht->has_dict[i], "join key %d: one side is a string column, the other is not", i);
    if (is_str) {
      cols.push_back(key_cols[i]);
      dicts.push_back(&ht->dict[i]);
    }
  }
  if (cols.empty()) return probe;
  encode_string_columns(probe, cols, &dicts, st, ev);
  return ev.view;
}

}  // namespace sb

using namespace sb;

extern "C" {

// filter == NULL: every row with non-NULL keys joins the relation.  Otherwise rows for which the predicate is not TRUE are left
// out (the FilterExec below the build side, fused: the filtered table is never materialised; payload columns are gathered from
// `build` by row id at probe time, so nothing else changes).
int sb_join_build_filtered(const sb_table *build, const int32_t *key_cols, int32_t nkeys, const sb_expr *filter, sb_stream *s,
                           sb_hash_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(build && key_cols && out, "null argument");
  cudaStream_t st = stream_of(s);
  int64_t n = build->nrows;
  SB_REQUIRE(n < 0xFFFFFFFFll, "build side has too many rows for one relation");
  SB_REQUIRE(nkeys >= 1 && nkeys <= JOIN_MAX_KEYS, "joins support 1..%d key columns (got %d)", JOIN_MAX_KEYS, nkeys);
  EncodedView ev;   // string key columns -> codes; the dictionaries move into the relation below
  {
    std::vector<int> scols;
    for (int i = 0; i < nkeys; i++)
      if (key_cols[i] >= 0 && key_cols[i] < (int)build->cols.size() && build->cols[key_cols[i]].type == SB_STRING) scols.push_back(key_cols[i]);
    if (!scols.empty()) encode_string_columns(build, scols, nullptr, st, ev);
  }
  JoinKeys k = make_join_keys(ev.view ? ev.view : build, key_cols, nkeys, nullptr);
  Scratch mask(filter ? n + 16 : 0, st);
  if (filter) eval_predicate(build, *filter, mask.as<uint8_t>(), st);   // validates the program even when n == 0
  sb_hash_table *ht = new sb_hash_table();
  ht->st = st;
  ht->nkeys = nkeys;
  ht->wide = k.wide;
  if (k.wide) {   // the key columns must outlive the build: keep the table they live in (the build table, or its encoded view)
    ht->key_table = ev.view ? ev.view : const_cast<sb_table *>(build);
    ht->key_table->refs.fetch_add(1);
    for (int i = 0; i < nkeys; i++) ht->key_table_col[i] = key_cols[i];
  }
  for (int i = 0; i < nkeys; i++) {
    if (const Column *d = ev.view ? ev.dictionary_of(key_cols[i]) : nullptr) {
      ht->has_dict[i] = true;
      ht->dict[i] = column_share(*d);
    }
    ht->key_col[i] = key_cols[i];
    ht->key_type[i] = k.type[i];
    ht->key_bits[i] = k.bits[i];
    ht->key_shift[i] = k.shift[i];
  }
  // size everything by what will actually be inserted: one pass over the keys (and the fused filter's mask)
  long long stats[4] = {0x7FFFFFFFFFFFFFFFll, -0x7FFFFFFFFFFFFFFFll - 1, 0, 0};
  if (n > 0) {
    Scratch dstats(32, st);
    SB_CUDA(cudaMemcpyAsync(dstats.ptr, stats, 32, cudaMemcpyHostToDevice, st));
    int64_t g = (n + JOIN_THREADS * 8 - 1) / (JOIN_THREADS * 8);
    if (g > (int64_t)rt().num_sms * 16) g = (int64_t)rt().num_sms * 16;
    build_stats_kernel<<<(unsigned)g, JOIN_THREADS, 0, st>>>(k, n, filter ? mask.as<uint8_t>() : nullptr, dstats.as<long long>());
    SB_LAUNCH_CHECK();
    SB_CUDA(cudaMemcpyAsync(stats, dstats.ptr, 32, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  const int64_t nin = stats[2];
  const bool ascending = !filter && nin == n && n > 0 && stats[3] == 0;   // strictly ascending, NULL-free: row = rank of the key
  ht->nkeys_in = nin;
  int64_t cap = 1024;
  while (cap < 2 * nin) cap <<= 1;
  ht->cap = cap;
  int64_t bwords = 1024;
  const uint64_t range = nin > 0 ? (uint64_t)stats[1] - (uint64_t)stats[0] + 1 : 0;
  // exact bitmap: dense keys, small ranges -- and SORTED sparse keys up to a 128 MB bitmap: keys that arrive in ascending order come
  // from a key-ordered scan, whose foreign-key side is usually clustered on the same key (lineitem by l_orderkey) and then walks the
  // bitmap sequentially, where a Bloom filter costs every streamed row a hash and a random L2 access (Q5's lineitem pass against
  // 4.6 M order keys spread over a range of 600 M)
  if (nin > 0 && range != 0 && range <= (1ull << 31) &&
      (range <= (1ull << 23) || range <= 64ull * (uint64_t)nin || (ascending && range <= (1ull << 30)))) {
    ht->exact = 1;
    ht->fmin = (uint64_t)stats[0];
    ht->frange = range;
    bwords = (int64_t)(range / 32 + 1);
  } else {
    while (bwords < nin && bwords < (8ll << 20)) bwords <<= 1;   // ~1 key per 32-bit word, at most 32 MB (L2-resident)
    ht->bloom_mask = (uint64_t)bwords - 1;
  }
  try {
    const unsigned nblocks = (unsigned)((n + JOIN_THREADS - 1) / JOIN_THREADS);
    const uint8_t *mask_dev = filter ? mask.as<uint8_t>() : nullptr;
    SB_CUDA(cudaMallocAsync((void **)&ht->null_key_flag, 8, st));   // [0] a NULL key was seen, [1] a key arrived twice
    SB_CUDA(cudaMemsetAsync(ht->null_key_flag, 0, 8, st));
    SB_CUDA(cudaMallocAsync((void **)&ht->bloom, (size_t)bwords * 4, st));
    SB_CUDA(cudaMemsetAsync(ht->bloom, 0, (size_t)bwords * 4, st));
    int32_t hflags[2] = {0, 0};
    bool built = false;
    if (ht->exact && range <= 8ull * (uint64_t)nin) {   // dense: try the direct-address table; a duplicate key voids the attempt
      SB_CUDA(cudaMallocAsync((void **)&ht->row_of, (size_t)range * 4, st));
      SB_CUDA(cudaMemsetAsync(ht->row_of, 0xff, (size_t)range * 4, st));
      {
        KernelTimer kt("join_build", st);
        join_build_kernel<<<nblocks, JOIN_THREADS, 0, st>>>(k, n, nullptr, cap, ht->null_key_flag, mask_dev, key_filter_of(ht));
        SB_LAUNCH_CHECK();
      }
      SB_CUDA(cudaMemcpyAsync(hflags, ht->null_key_flag, 8, cudaMemcpyDeviceToHost, st));
      SB_CUDA(cudaStreamSynchronize(st));
      if (!hflags[1]) {
        built = true;
        ht->unique = 1;
      } else {
        cudaFreeAsync(ht->row_of, st);
        ht->row_of = nullptr;
        SB_CUDA(cudaMemsetAsync(ht->bloom, 0, (size_t)bwords * 4, st));
        SB_CUDA(cudaMemsetAsync(ht->null_key_flag, 0, 8, st));
      }
    }
    if (!built && ht->exact && ascending) {   // sorted mode: bitmap + rank prefix, no slot table
      {
        KernelTimer kt("join_build", st);
        join_build_kernel<<<nblocks, JOIN_THREADS, 0, st>>>(k, n, nullptr, cap, ht->null_key_flag, mask_dev, key_filter_of(ht));
        SB_LAUNCH_CHECK();
        Scratch pc(bwords * 4 + 16, st);
        SB_CUDA(cudaMallocAsync((void **)&ht->rank, (size_t)bwords * 4 + 16, st));
        word_popc_kernel<<<(unsigned)((bwords + 255) / 256), 256, 0, st>>>(ht->bloom, bwords, pc.as<int32_t>());
        SB_LAUNCH_CHECK();
        exclusive_scan_i32(pc.as<int32_t>(), (int32_t *)ht->rank, bwords, nullptr, st);
      }
      ht->unique = 1;
      built = true;
    }
    if (!built) {
      SB_CUDA(cudaMallocAsync((void **)&ht->slots, (size_t)cap * sizeof(JoinSlot), st));
      SB_CUDA(cudaMemsetAsync(ht->slots, 0xff, (size_t)cap * sizeof(JoinSlot), st));
      if (n > 0) {
        KernelTimer kt("join_build", st);
        join_build_kernel<<<nblocks, JOIN_THREADS, 0, st>>>(k, n, ht->slots, cap, ht->null_key_flag, mask_dev, key_filter_of(ht));
        SB_LAUNCH_CHECK();
      }
      if (ht->exact) {   // unique keys? (the answer picks the probe strategy, so it is worth one round trip here)
        SB_CUDA(cudaMemcpyAsync(hflags, ht->null_key_flag, 8, cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));
        ht->unique = hflags[1] ? 0 : 1;
      }
    }
    ht->build = const_cast<sb_table *>(build);
    ht->build->refs.fetch_add(1);
    // a relation is handed to other task threads / streams (broadcast): instead of draining the stream here, the build leaves an
    // event behind and every consumer on another stream waits for it on the device (wait_relation)
    SB_CUDA(cudaEventCreateWithFlags(&ht->ready, cudaEventDisableTiming));
    SB_CUDA(cudaEventRecord(ht->ready, st));
  } catch (...) {
    if (ht->slots) cudaFreeAsync(ht->slots, st);
    if (ht->null_key_flag) cudaFreeAsync(ht->null_key_flag, st);
    if (ht->bloom) cudaFreeAsync(ht->bloom, st);
    if (ht->row_of) cudaFreeAsync(ht->row_of, st);
    if (ht->rank) cudaFreeAsync(ht->rank, st);
    if (ht->ready) cudaEventDestroy(ht->ready);
    if (ht->key_table && ht->key_table->refs.fetch_sub(1) == 1) table_free(ht->key_table);
    for (int i = 0; i < 4; i++)
      if (ht->has_dict[i]) column_release(ht->dict[i]);
    delete ht;
    throw;
  }
  *out = ht;
  SB_API_END
}

int sb_join_build(const sb_table *build, const int32_t *key_cols, int32_t nkeys, sb_stream *s, sb_hash_table **out) {
  return sb_join_build_filtered(build, key_cols, nkeys, nullptr, s, out);
}

int sb_hash_table_release(sb_hash_table *ht) {
  SB_API_BEGIN
  if (ht) {
    if (ht->slots) cudaFreeAsync(ht->slots, ht->st);
    if (ht->null_key_flag) cudaFreeAsync(ht->null_key_flag, ht->st);
    if (ht->bloom) cudaFreeAsync(ht->bloom, ht->st);
    if (ht->row_of) cudaFreeAsync(ht->row_of, ht->st);
    if (ht->rank) cudaFreeAsync(ht->rank, ht->st);
    if (ht->ready) cudaEventDestroy(ht->ready);
    if (ht->key_table && ht->key_table->refs.fetch_sub(1) == 1) table_free(ht->key_table);
    if (ht->build && ht->build->refs.fetch_sub(1) == 1) table_free(ht->build);
    for (int i = 0; i < 4; i++)
      if (ht->has_dict[i]) column_release(ht->dict[i]);
    delete ht;
  }
  SB_API_END
}

__global__ void exists_kernel(const uint32_t *__restrict__ first, int64_t n, uint8_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = first[i] != sb::FREE_SLOT;
}
__global__ void unmatched_kernel(const uint8_t *__restrict__ matched, int64_t n, uint8_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = !matched[i];
}
__global__ void fill_i64_kernel(int64_t *out, int64_t n, int64_t v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

// device-side ordering between a relation's build and a consumer on another stream (same stream: already ordered)
static void wait_relation(const sb_hash_table *ht, cudaStream_t st) {
  if (ht->ready && st != ht->st) SB_CUDA(cudaStreamWaitEvent(st, ht->ready, 0));
}

// a zero-copy view of `t` restricted to `cols` (NULL: all columns); the caller frees it with table_free
static sb_table *column_view(const sb_table *t, const int32_t *cols, int32_t ncols) {
  sb_table *v = table_new(t->nrows);
  if (!cols) {
    for (auto &c : t->cols) v->cols.push_back(column_share(c));
    return v;
  }
  for (int i = 0; i < ncols; i++) {
    if (cols[i] < 0 || cols[i] >= (int)t->cols.size()) {
      table_free(v);
      fail(SB_ERR_INVALID, "join output column %d out of range", cols[i]);
    }
    v->cols.push_back(column_share(t->cols[cols[i]]));
  }
  return v;
}
struct TableGuard {
  sb_table *t;
  ~TableGuard() { if (t) sb::table_free(t); }
};

int sb_join_probe(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys, int32_t join_type,
                  sb_stream *s, sb_table **out) {
  return sb_join_probe_ex(ht, probe, key_cols, nkeys, join_type, nullptr, s, out);
}

int sb_join_probe_ex(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys, int32_t join_type,
                     const sb_join_options *opt, sb_stream *s, sb_table **out) {
  if (opt && opt->condition) {
    if (opt->probe_filter || opt->probe_out_cols || opt->build_out_cols || opt->n_runtime_filters > 0) {
      sb::set_last_error("sb_join_probe_ex: a residual condition cannot be combined with a fused filter / projection / runtime filter yet");
      return SB_ERR_UNSUPPORTED;
    }
    return sb_join_probe_condition(ht, probe, key_cols, nkeys, join_type, opt->condition, s, out);
  }
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(ht && probe && key_cols && out, "null argument");
  const sb_expr *probe_filter = opt ? opt->probe_filter : nullptr;
  // the views the output columns are gathered from: the fused ProjectExec above the join keeps only what the plan needs
  TableGuard probe_view{column_view(probe, opt ? opt->probe_out_cols : nullptr, opt ? opt->n_probe_out : 0)};
  TableGuard build_view{column_view(ht->build, opt ? opt->build_out_cols : nullptr, opt ? opt->n_build_out : 0)};
  SB_REQUIRE(nkeys == ht->nkeys, "probe has %d key columns, the relation was built on %d", nkeys, ht->nkeys);
  SB_REQUIRE(join_type >= SB_JOIN_INNER && join_type <= SB_JOIN_LEFT_ANTI_NULL_AWARE, "unknown join type %d", join_type);
  cudaStream_t st = stream_of(s);
  wait_relation(ht, st);
  const int64_t n = probe->nrows, nbuild = ht->build->nrows;
  EncodedView key_view;
  JoinKeys k = make_join_keys(probe_key_source(ht, probe, key_cols, nkeys, st, key_view), key_cols, nkeys, ht);
  // the kernels know inner / streamed-outer / semi / anti / existence; the build-side-preserving joins are those plus the build
  // rows nobody matched (ShuffledHashJoinExec.buildSideOrFullOuterJoin, SQLX/joins/ShuffledHashJoinExec.scala:130-330)
  const bool build_rows_too = join_type == SB_JOIN_FULL_OUTER || join_type == SB_JOIN_BUILD_OUTER;
  int kt_type = join_type;
  if (join_type == SB_JOIN_FULL_OUTER) kt_type = SB_JOIN_LEFT_OUTER;
  if (join_type == SB_JOIN_BUILD_OUTER) kt_type = SB_JOIN_INNER;
  int null_aware = 0;
  if (join_type == SB_JOIN_LEFT_ANTI_NULL_AWARE) {
    // BroadcastHashJoinExec.scala:137-162: empty relation -> every streamed row; a NULL key in the relation -> no row;
    // otherwise streamed rows with a NULL key are dropped and the rest is an anti join
    SB_REQUIRE(nkeys == 1, "the null-aware anti join takes a single key (NOT IN subquery)");
    kt_type = SB_JOIN_LEFT_ANTI;
    int32_t flag = 0;
    SB_CUDA(cudaMemcpyAsync(&flag, ht->null_key_flag, 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    if (probe_filter) fail(SB_ERR_UNSUPPORTED, "null-aware anti join with a fused filter");
    if (nbuild == 0) {
      sb_table *t = table_new(n);
      for (auto &c : probe_view.t->cols) t->cols.push_back(column_share(c));
      *out = t;
      return SB_OK;
    }
    if (flag) {
      Scratch none(16, st);
      *out = gather_table(probe_view.t, none.as<int64_t>(), 0, false, st);
      return SB_OK;
    }
    null_aware = 1;
  }
  const bool pairs = kt_type == SB_JOIN_INNER || kt_type == SB_JOIN_LEFT_OUTER;
  unsigned nb = (unsigned)((n + JOIN_THREADS - 1) / JOIN_THREADS);
  Scratch total(16, st);
  Scratch matched(build_rows_too ? nbuild + 16 : 0, st);
  if (build_rows_too) SB_CUDA(cudaMemsetAsync(matched.ptr, 0, (size_t)nbuild + 16, st));
  // candidate list (see join_candidate_kernel): worth its pass when the streamed side is long
  const bool use_cand = n >= (1 << 20) && join_type != SB_JOIN_EXISTENCE;
  const KeyFilter kf = key_filter_of(ht);
  // what the candidate pass can settle by itself.  Behind an EXACT prefilter a candidate is a row whose key is in the relation, so
  // semi / anti joins are finished by the pass, and with unique keys inner / outer joins need one lookup per candidate
  // (no count / scan / fill).
  const bool settled = use_cand && ht->exact && !build_rows_too &&
                       (kt_type == SB_JOIN_LEFT_SEMI || kt_type == SB_JOIN_LEFT_ANTI || (ht->unique && pairs));
  int cand_mode = kt_type == SB_JOIN_INNER || kt_type == SB_JOIN_LEFT_SEMI ? CAND_PRESENT : CAND_ALL;
  if (settled && kt_type == SB_JOIN_LEFT_ANTI) cand_mode = null_aware ? CAND_ABSENT_KEYED : CAND_ABSENT;
  // the FilterExec below the streamed side, fused: rows failing it are not part of the input.  A conjunction of column-vs-literal
  // comparisons is evaluated inside the candidate pass itself; anything else becomes a byte mask first.
  SimplePred sp;
  sp.nterms = 0;
  bool pred_in_pass = false;
  if (probe_filter) {
    expr_validate(probe, *probe_filter);
    pred_in_pass = use_cand && !config().expr_interpret_only && match_simple_predicate(probe, *probe_filter, sp);
    if (!pred_in_pass) sp.nterms = 0;
  }
  // runtime filters (InjectRuntimeFilter): on the candidate list after the pass when there is one, else folded into the byte mask
  std::vector<JoinKeys> rf_keys;
  std::vector<KeyFilter> rf_filters;
  if (opt && opt->n_runtime_filters > 0) {
    SB_REQUIRE(opt->runtime_filter_cols && opt->runtime_filter_relations, "runtime filters: null argument");
    if (!(join_type == SB_JOIN_INNER || join_type == SB_JOIN_LEFT_SEMI))
      fail(SB_ERR_UNSUPPORTED, "runtime filters drop streamed rows: only inner and left semi joins take them");
    for (int i = 0; i < opt->n_runtime_filters; i++) {
      const sb_hash_table *r = opt->runtime_filter_relations[i];
      SB_REQUIRE(r, "runtime filter %d: null relation", i);
      wait_relation(r, st);
      if (r->nkeys != 1 || r->wide || r->has_dict[0]) fail(SB_ERR_UNSUPPORTED, "runtime filter %d: the creation side must be a relation on one fixed-width key", i);
      if (!r->bloom) continue;   // a relation without a prefilter: the filter is an optimisation, leaving it out changes nothing
      const int32_t c = opt->runtime_filter_cols[i];
      SB_REQUIRE(c >= 0 && c < (int)probe->cols.size(), "runtime filter %d: column %d out of range", i, c);
      const int32_t ct = probe->cols[c].type;
      if (ct == SB_STRING || ct == SB_DECIMAL128 || type_width(ct) * 8 != r->key_bits[0]) continue;   // differently packed: leave the filter out
      rf_keys.push_back(make_join_keys(probe, &c, 1, r));
      rf_filters.push_back(key_filter_of(r));
    }
  }
  const bool rf_post = !rf_keys.empty() && use_cand && cand_mode == CAND_PRESENT;   // on the candidate list, after the pass
  const bool rf_mask = !rf_keys.empty() && !rf_post;
  const bool pred_mask = probe_filter && !pred_in_pass;
  Scratch pmask(pred_mask || rf_mask ? n + 16 : 0, st);
  if (pred_mask && n > 0) eval_predicate(probe, *probe_filter, pmask.as<uint8_t>(), st);
  if (rf_mask && n > 0)
    for (size_t i = 0; i < rf_keys.size(); i++) {
      runtime_filter_mask_kernel<<<(unsigned)((n + JOIN_THREADS - 1) / JOIN_THREADS), JOIN_THREADS, 0, st>>>(rf_keys[i], n, rf_filters[i], pmask.as<uint8_t>(),
                                                                                                     pred_mask || i > 0 ? 1 : 0);
      SB_LAUNCH_CHECK();
    }
  const uint8_t *pmask_dev = pred_mask || rf_mask ? pmask.as<uint8_t>() : nullptr;
  int64_t nitems = n;
  std::unique_ptr<Scratch> cand_rows;
  if (use_cand) {
    KernelTimer kt("join_candidates", st);
    const int64_t nwords = (n + CAND_ROWS - 1) / CAND_ROWS;
    const unsigned cb = (unsigned)((n + CAND_TILE - 1) / CAND_TILE);
    Scratch bits(nwords * 2 + 16, st), bcount((int64_t)cb * 4 + 16, st), boff((int64_t)cb * 8 + 16, st), tot(8, st);
    const int fast_key = k.n == 1 && !k.valid[0] && k.type[0] != SB_FLOAT32 && k.type[0] != SB_FLOAT64 && k.type[0] != SB_BOOL &&
                         ((uintptr_t)k.data[0] & 15) == 0;
    if (config().join_cand >= 1) {
      // the ballot words are written as uint32: the buffer must hold whole 32-row words (nwords is in 16-row units)
      const bool int_key = k.n == 1 && !k.valid[0] && k.type[0] != SB_FLOAT32 && k.type[0] != SB_FLOAT64 && k.type[0] != SB_BOOL;
      const int kw = !int_key ? 0 : (k.bits[0] == 64 ? 8 : k.bits[0] == 32 ? 4 : 0);
      uint32_t *bo = bits.as<uint32_t>();
      int32_t *bc = bcount.as<int32_t>();
#define SB_CAND(KW, STEP, MINB) join_candidate_strided_kernel<KW, STEP, MINB><<<cb, JOIN_THREADS, 0, st>>>(k, n, sp, pmask_dev, kf, cand_mode, bo, bc)
      const int v = config().join_cand;   // 1: 8 rows per lane and step; 2: 4 rows, 4 blocks / SM; 3: 8 rows, 3 blocks / SM
      if (v == 2) { if (kw == 8) SB_CAND(8, 4, 4); else if (kw == 4) SB_CAND(4, 4, 4); else SB_CAND(0, 4, 4); }
      else if (v == 3) { if (kw == 8) SB_CAND(8, 8, 3); else if (kw == 4) SB_CAND(4, 8, 3); else SB_CAND(0, 8, 3); }
      else { if (kw == 8) SB_CAND(8, 8, 1); else if (kw == 4) SB_CAND(4, 8, 1); else SB_CAND(0, 8, 1); }
#undef SB_CAND
    } else {
      join_candidate_kernel<<<cb, JOIN_THREADS, 0, st>>>(k, n, sp, pmask_dev, kf, cand_mode, fast_key, bits.as<uint16_t>(), bcount.as<int32_t>());
    }
    SB_LAUNCH_CHECK();
    exclusive_scan_i32_to_i64(bcount.as<int32_t>(), boff.as<int64_t>(), cb, tot.as<int64_t>(), st);
    SB_CUDA(cudaMemcpyAsync(&nitems, tot.ptr, 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    cand_rows.reset(new Scratch(nitems * 8 + 16, st));
    if (nitems > 0) {
      candidate_rows_kernel<<<cb, JOIN_THREADS, 0, st>>>(bits.as<uint16_t>(), nwords, boff.as<int64_t>(), cand_rows->as<int64_t>());
      SB_LAUNCH_CHECK();
    }
    if (rf_post && nitems > 0) {   // runtime filters over the candidate list: flags -> compaction -> the surviving rows, still in row order
      Scratch flags(nitems + 16, st), idx(nitems * 8 + 16, st);
      const unsigned fb = (unsigned)((nitems + JOIN_THREADS - 1) / JOIN_THREADS);
      for (size_t i = 0; i < rf_keys.size(); i++) {
        runtime_filter_rows_kernel<<<fb, JOIN_THREADS, 0, st>>>(rf_keys[i], cand_rows->as<int64_t>(), nitems, rf_filters[i], flags.as<uint8_t>(), i > 0 ? 1 : 0);
        SB_LAUNCH_CHECK();
      }
      const int64_t m = compact_mask(flags.as<uint8_t>(), nitems, idx.as<int64_t>(), st);
      std::unique_ptr<Scratch> kept(new Scratch(m * 8 + 16, st));
      if (m > 0) {
        take_rows_kernel<<<(unsigned)((m + JOIN_THREADS - 1) / JOIN_THREADS), JOIN_THREADS, 0, st>>>(cand_rows->as<int64_t>(), idx.as<int64_t>(), m, kept->as<int64_t>());
        SB_LAUNCH_CHECK();
      }
      cand_rows = std::move(kept);
      nitems = m;
    }
    nb = (unsigned)((nitems + JOIN_THREADS - 1) / JOIN_THREADS);
  }
  const int64_t *rows = use_cand ? cand_rows->as<int64_t>() : nullptr;
  if (settled) {
    // the candidate list IS the streamed half of the output; partners (inner / outer) come from one lookup each
    const int64_t nout = nitems;
    Scratch out_build(pairs ? nout * 8 + 16 : 0, st);
    if (pairs && nout > 0) {
      KernelTimer kt("join_probe", st);
      join_lookup_kernel<<<nb, JOIN_THREADS, 0, st>>>(k, rows, nout, ht->slots, ht->cap, kf, kt_type == SB_JOIN_LEFT_OUTER ? 1 : 0, out_build.as<int64_t>());
      SB_LAUNCH_CHECK();
    }
    // every streamed row a candidate: the streamed half of the output is the input (shared buffers, no gather)
    const bool identity = nout == n;
    auto take_streamed = [&](const Column &c) { return identity ? column_share(c) : gather_column(c, rows, nout, false, st); };
    sb_table *left = nullptr;
    if (identity) {
      left = table_new(n);
      for (auto &c : probe_view.t->cols) left->cols.push_back(column_share(c));
    } else {
      left = gather_table(probe_view.t, rows, nout, false, st);
    }
    if (pairs) {
      // inner join: a build-side KEY column of the output holds, row for row, the values of the streamed side's key column
      // (integer keys of one type compare equal only when they are the same bits), so it is taken from there -- a sequential
      // read instead of a random gather over the build table
      const int nb_cols = (int)build_view.t->cols.size();
      std::vector<int> from_streamed(nb_cols, -1);
      std::vector<Column> keyed;
      sb_table *rest = table_new(ht->build->nrows);
      sb_table *right = nullptr;
      try {
        for (int j = 0; j < nb_cols; j++) {
          const int bj = opt && opt->build_out_cols ? opt->build_out_cols[j] : j;
          if (kt_type == SB_JOIN_INNER)
            for (int i = 0; i < nkeys; i++) {
              const Column &pc = probe->cols[key_cols[i]];
              const int32_t t = ht->build->cols[bj].type;
              if (ht->key_col[i] == bj && !ht->has_dict[i] && pc.type == t && t != SB_FLOAT32 && t != SB_FLOAT64 && t != SB_STRING) from_streamed[j] = key_cols[i];
            }
          if (from_streamed[j] < 0) rest->cols.push_back(column_share(build_view.t->cols[j]));
        }
        right = gather_table(rest, out_build.as<int64_t>(), nout, kt_type == SB_JOIN_LEFT_OUTER, st);
        for (int j = 0; j < nb_cols; j++) {
          if (from_streamed[j] < 0) continue;
          const Column &bc = ht->build->cols[opt && opt->build_out_cols ? opt->build_out_cols[j] : j];
          Column c = take_streamed(probe->cols[from_streamed[j]]);
          c.type = bc.type;
          c.scale = bc.scale;
          keyed.push_back(c);
        }
      } catch (...) {
        for (auto &c : keyed) column_release(c);
        table_free(rest);
        if (right) table_free(right);
        table_free(left);
        throw;
      }
      size_t next = 0, next_keyed = 0;   // nothing below throws
      for (int j = 0; j < nb_cols; j++) left->cols.push_back(from_streamed[j] >= 0 ? keyed[next_keyed++] : right->cols[next++]);
      right->cols.clear();
      table_free(rest);
      table_free(right);
    }
    *out = left;
    return SB_OK;
  }
  Scratch counts(nitems * 4 + 16, st), first(nitems * 4 + 16, st), block_counts((int64_t)nb * 4 + 16, st), offsets((int64_t)nb * 8 + 16, st);
  if (nitems > 0) {
    KernelTimer kt("join_probe", st);
    join_count_kernel<<<nb, JOIN_THREADS, 0, st>>>(k, nitems, ht->slots, ht->cap, kt_type, null_aware, counts.as<int32_t>(), first.as<uint32_t>(),
                                                   block_counts.as<int32_t>(), build_rows_too ? matched.as<uint8_t>() : nullptr,
                                                   use_cand ? nullptr : pmask_dev, kf, rows, build_side_keys(ht));
    SB_LAUNCH_CHECK();
  }
  if (join_type == SB_JOIN_EXISTENCE) {   // HashJoin.existenceJoin :301: the streamed row plus one boolean
    if (probe_filter) fail(SB_ERR_UNSUPPORTED, "the existence join keeps every streamed row: filter the streamed side before it");
    sb_table *t = table_new(n);
    try {
      for (auto &c : probe_view.t->cols) t->cols.push_back(column_share(c));
      Column e = column_alloc(SB_BOOL, 0, n, false, st);
      t->cols.push_back(e);
      if (n > 0) {
        exists_kernel<<<nb, JOIN_THREADS, 0, st>>>(first.as<uint32_t>(), n, (uint8_t *)e.data->ptr);
        SB_LAUNCH_CHECK();
      }
    } catch (...) {
      table_free(t);
      throw;
    }
    *out = t;
    return SB_OK;
  }
  exclusive_scan_i32_to_i64(block_counts.as<int32_t>(), offsets.as<int64_t>(), nb, total.as<int64_t>(), st);
  // build rows without a partner, in build order (their count comes back with the pair count: one host round trip)
  Scratch un_mask(build_rows_too ? nbuild + 16 : 0, st), un_idx(build_rows_too ? nbuild * 8 + 16 : 0, st),
      un_f32(build_rows_too ? compact_tiles(nbuild) * 4 + 16 : 0, st), un_pos(build_rows_too ? compact_tiles(nbuild) * 8 + 16 : 0, st);
  if (build_rows_too) {
    if (nbuild > 0) {
      unmatched_kernel<<<(unsigned)((nbuild + 255) / 256), 256, 0, st>>>(matched.as<uint8_t>(), nbuild, un_mask.as<uint8_t>());
      SB_LAUNCH_CHECK();
      compact_mask_async(un_mask.as<uint8_t>(), nbuild, un_idx.as<int64_t>(), un_f32.as<int32_t>(), un_pos.as<int64_t>(), total.as<int64_t>() + 1, st);
    } else SB_CUDA(cudaMemsetAsync(total.as<int64_t>() + 1, 0, 8, st));
  }
  int64_t totals[2] = {0, 0};
  SB_CUDA(cudaMemcpyAsync(totals, total.ptr, build_rows_too ? 16 : 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  const int64_t npairs = totals[0], nun = build_rows_too ? totals[1] : 0, nout = npairs + nun;
  Scratch out_probe(nout * 8 + 16, st), out_build(pairs ? nout * 8 + 16 : 0, st);
  if (nitems > 0 && npairs > 0) {
    KernelTimer kt("join_fill", st);
    join_fill_kernel<<<nb, JOIN_THREADS, 0, st>>>(k, nitems, ht->slots, ht->cap, kt_type, counts.as<int32_t>(),
                                                  offsets.as<int64_t>(), first.as<uint32_t>(), out_probe.as<int64_t>(),
                                                  pairs ? out_build.as<int64_t>() : nullptr, rows, build_side_keys(ht));
    SB_LAUNCH_CHECK();
  }
  if (nun > 0) {
    fill_i64_kernel<<<(unsigned)((nun + 255) / 256), 256, 0, st>>>(out_probe.as<int64_t>() + npairs, nun, -1);
    SB_LAUNCH_CHECK();
    SB_CUDA(cudaMemcpyAsync(out_build.as<int64_t>() + npairs, un_idx.ptr, (size_t)nun * 8, cudaMemcpyDeviceToDevice, st));
  }
  sb_table *left = gather_table(probe_view.t, out_probe.as<int64_t>(), nout, build_rows_too, st);
  if (!pairs) {
    *out = left;
  } else {
    sb_table *right = nullptr;
    try {
      right = gather_table(build_view.t, out_build.as<int64_t>(), nout, kt_type == SB_JOIN_LEFT_OUTER, st);
    } catch (...) {
      table_free(left);
      throw;
    }
    for (auto &c : right->cols) left->cols.push_back(c);   // output = streamed columns ++ build columns (HashJoin.scala:55-70)
    right->cols.clear();
    table_free(right);
    *out = left;
  }
  SB_API_END
}

__global__ void scatter_flag_kernel(const int64_t *__restrict__ idx, int64_t n, uint8_t *__restrict__ flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && idx[i] >= 0) flags[idx[i]] = 1;
}
__global__ void invert_flag_kernel(uint8_t *flags, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = !flags[i];
}
__global__ void gather_i64_kernel(const int64_t *__restrict__ src, const int64_t *__restrict__ idx, int64_t n, int64_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}
__global__ void null_key_rows_kernel(sb::JoinKeys k, int64_t n, uint8_t *__restrict__ flags) {   // flags[i] = 1 where the key is NULL
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t key;
  if (i < n) flags[i] = !sb::join_key(k, i, key);
}

// Equi-join with a residual condition (HashJoin.scala:144-172 boundCondition): `condition` is evaluated on the joined row
// (streamed columns ++ build columns) of every key match, and only pairs for which it is TRUE count as matches -- which matters
// for every join type but inner: an outer row whose key matches but whose condition never holds is NULL-extended, a semi / anti /
// existence row is judged by the surviving pairs.  condition == NULL is sb_join_probe.
int sb_join_probe_condition(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys, int32_t join_type,
                            const sb_expr *condition, sb_stream *s, sb_table **out) {
  if (!condition) return sb_join_probe(ht, probe, key_cols, nkeys, join_type, s, out);
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(ht && probe && key_cols && out, "null argument");
  SB_REQUIRE(join_type >= SB_JOIN_INNER && join_type <= SB_JOIN_LEFT_ANTI_NULL_AWARE, "unknown join type %d", join_type);
  if (join_type == SB_JOIN_LEFT_ANTI_NULL_AWARE) fail(SB_ERR_UNSUPPORTED, "the null-aware anti join takes no residual condition (BroadcastHashJoinExec.scala:73-76)");
  cudaStream_t st = stream_of(s);
  const int64_t n = probe->nrows, nbuild = ht->build->nrows;
  // 1. every key match as an inner pair table
  sb_table *pairs_tbl = nullptr;
  {
    int rc = sb_join_probe(ht, probe, key_cols, nkeys, SB_JOIN_INNER, s, &pairs_tbl);
    if (rc != SB_OK) fail(rc, "%s", sb_last_error());
  }
  // the pair indices are needed as well: recompute them cheaply by joining row-id columns would double the work, so the pair table
  // is built again below from indices; here only the mask is taken from it
  struct Guard { sb_table *&t; ~Guard() { if (t) sb::table_free(t); } } g1{pairs_tbl};
  const int64_t npairs = pairs_tbl->nrows;
  Scratch mask(npairs + 16, st);
  eval_predicate(pairs_tbl, *condition, mask.as<uint8_t>(), st);   // validates the program even when there is no pair
  // pair indices: the same kernels again with index outputs only (count + fill), cheaper than carrying row ids through the gather
  EncodedView key_view;
  JoinKeys k = make_join_keys(probe_key_source(ht, probe, key_cols, nkeys, st, key_view), key_cols, nkeys, ht);
  unsigned nb = (unsigned)((n + JOIN_THREADS - 1) / JOIN_THREADS);
  Scratch counts(n * 4 + 16, st), first(n * 4 + 16, st), block_counts((int64_t)nb * 4 + 16, st), offsets((int64_t)nb * 8 + 16, st), total(8, st);
  Scratch pi(npairs * 8 + 16, st), bi(npairs * 8 + 16, st);
  if (n > 0) {
    join_count_kernel<<<nb, JOIN_THREADS, 0, st>>>(k, n, ht->slots, ht->cap, SB_JOIN_INNER, 0, counts.as<int32_t>(), first.as<uint32_t>(),
                                                   block_counts.as<int32_t>(), nullptr, nullptr, key_filter_of(ht), nullptr, build_side_keys(ht));
    SB_LAUNCH_CHECK();
    exclusive_scan_i32_to_i64(block_counts.as<int32_t>(), offsets.as<int64_t>(), nb, total.as<int64_t>(), st);
    if (npairs > 0) {
      join_fill_kernel<<<nb, JOIN_THREADS, 0, st>>>(k, n, ht->slots, ht->cap, SB_JOIN_INNER, counts.as<int32_t>(), offsets.as<int64_t>(),
                                                    first.as<uint32_t>(), pi.as<int64_t>(), bi.as<int64_t>(), nullptr, build_side_keys(ht));
      SB_LAUNCH_CHECK();
    }
  }
  // 2. surviving pairs
  Scratch keep(npairs * 8 + 16, st);
  const int64_t nkeep = npairs > 0 ? compact_mask(mask.as<uint8_t>(), npairs, keep.as<int64_t>(), st) : 0;
  Scratch spi(nkeep * 8 + 16, st), sbi(nkeep * 8 + 16, st);
  if (nkeep > 0) {
    gather_i64_kernel<<<(unsigned)((nkeep + 255) / 256), 256, 0, st>>>(pi.as<int64_t>(), keep.as<int64_t>(), nkeep, spi.as<int64_t>());
    gather_i64_kernel<<<(unsigned)((nkeep + 255) / 256), 256, 0, st>>>(bi.as<int64_t>(), keep.as<int64_t>(), nkeep, sbi.as<int64_t>());
    SB_LAUNCH_CHECK();
  }
  // 3. which streamed / build rows have a surviving pair
  Scratch pflag(n + 16, st), bflag(nbuild + 16, st);
  SB_CUDA(cudaMemsetAsync(pflag.ptr, 0, (size_t)n + 16, st));
  SB_CUDA(cudaMemsetAsync(bflag.ptr, 0, (size_t)nbuild + 16, st));
  if (nkeep > 0) {
    scatter_flag_kernel<<<(unsigned)((nkeep + 255) / 256), 256, 0, st>>>(spi.as<int64_t>(), nkeep, pflag.as<uint8_t>());
    scatter_flag_kernel<<<(unsigned)((nkeep + 255) / 256), 256, 0, st>>>(sbi.as<int64_t>(), nkeep, bflag.as<uint8_t>());
    SB_LAUNCH_CHECK();
  }
  auto rows_where = [&](Scratch &flags, int64_t rows, bool want_set, Scratch &idx_out) -> int64_t {
    if (rows == 0) return 0;
    if (!want_set) {
      invert_flag_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(flags.as<uint8_t>(), rows);
      SB_LAUNCH_CHECK();
    }
    return compact_mask(flags.as<uint8_t>(), rows, idx_out.as<int64_t>(), st);
  };
  if (join_type == SB_JOIN_EXISTENCE) {
    sb_table *t = table_new(n);
    for (auto &c : probe->cols) t->cols.push_back(column_share(c));
    Column e = column_alloc(SB_BOOL, 0, n, false, st);
    t->cols.push_back(e);
    if (n > 0) SB_CUDA(cudaMemcpyAsync(e.data->ptr, pflag.ptr, (size_t)n, cudaMemcpyDeviceToDevice, st));
    *out = t;
    SB_CUDA(cudaStreamSynchronize(st));
    return SB_OK;
  }
  if (join_type == SB_JOIN_LEFT_SEMI || join_type == SB_JOIN_LEFT_ANTI) {
    Scratch idx(n * 8 + 16, st);
    const int64_t m = rows_where(pflag, n, join_type == SB_JOIN_LEFT_SEMI, idx);
    *out = gather_table(probe, idx.as<int64_t>(), m, false, st);
    SB_CUDA(cudaStreamSynchronize(st));
    return SB_OK;
  }
  const bool keep_probe = join_type == SB_JOIN_LEFT_OUTER || join_type == SB_JOIN_FULL_OUTER;
  const bool keep_build = join_type == SB_JOIN_BUILD_OUTER || join_type == SB_JOIN_FULL_OUTER;
  Scratch up(keep_probe ? n * 8 + 16 : 0, st), ub(keep_build ? nbuild * 8 + 16 : 0, st);
  const int64_t nup = keep_probe ? rows_where(pflag, n, false, up) : 0;
  const int64_t nub = keep_build ? rows_where(bflag, nbuild, false, ub) : 0;
  const int64_t nout = nkeep + nup + nub;
  Scratch op(nout * 8 + 16, st), ob(nout * 8 + 16, st);
  if (nkeep > 0) {
    SB_CUDA(cudaMemcpyAsync(op.ptr, spi.ptr, (size_t)nkeep * 8, cudaMemcpyDeviceToDevice, st));
    SB_CUDA(cudaMemcpyAsync(ob.ptr, sbi.ptr, (size_t)nkeep * 8, cudaMemcpyDeviceToDevice, st));
  }
  if (nup > 0) {
    SB_CUDA(cudaMemcpyAsync(op.as<int64_t>() + nkeep, up.ptr, (size_t)nup * 8, cudaMemcpyDeviceToDevice, st));
    fill_i64_kernel<<<(unsigned)((nup + 255) / 256), 256, 0, st>>>(ob.as<int64_t>() + nkeep, nup, -1);
    SB_LAUNCH_CHECK();
  }
  if (nub > 0) {
    fill_i64_kernel<<<(unsigned)((nub + 255) / 256), 256, 0, st>>>(op.as<int64_t>() + nkeep + nup, nub, -1);
    SB_LAUNCH_CHECK();
    SB_CUDA(cudaMemcpyAsync(ob.as<int64_t>() + nkeep + nup, ub.ptr, (size_t)nub * 8, cudaMemcpyDeviceToDevice, st));
  }
  sb_table *left = gather_table(probe, op.as<int64_t>(), nout, keep_build, st);
  sb_table *right = nullptr;
  try {
    right = gather_table(ht->build, ob.as<int64_t>(), nout, keep_probe, st);
  } catch (...) {
    table_free(left);
    throw;
  }
  for (auto &c : right->cols) left->cols.push_back(c);
  right->cols.clear();
  table_free(right);
  *out = left;
  SB_CUDA(cudaStreamSynchronize(st));
  SB_API_END
}

}  // extern "C"
