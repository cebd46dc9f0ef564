// window.cu -- WindowExec (sql/core/src/main/scala/org/apache/spark/sql/execution/window/WindowExec.scala:90,
// WindowEvaluatorFactoryBase.scala, WindowFunctionFrame.scala) on the GPU.
//
// The reference requires its child sorted by partitionSpec ++ orderSpec, walks one partition at a time and evaluates every
// window expression through a frame object (whole partition / growing / shrinking / sliding / offset).  Here:
//   1. rows are sorted by (partition keys ASC NULLS FIRST, order spec) with the stable radix sort of sort.cu -- the output
//      order of the reference;
//   2. one pass marks partition heads and peer-group heads (adjacent-row comparison with grouping equality: NULL = NULL,
//      NaN = NaN, -0.0 = 0.0; string columns through their dictionary codes);
//   3. heads -> dense ids (prefix sums) -> first row of every partition / peer group (scatter), so each row knows
//      [seg_start, seg_end) and [peer_start, peer_end);
//   4. every function is a per-row formula over those bounds and over SEGMENTED inclusive scans of its input (sum / count /
//      min / max restart at partition heads): a frame [lo, hi] of a row is turned into S[hi] - S[lo - 1] (count, integer sum),
//      +0.0 + S[hi] (double sum / avg of a frame that starts at the partition's first row), +0.0 + the aligned block sums inside
//      [lo, hi] (any other double sum / avg: the result depends on the frame's own rows only, so an inf, NaN or 1e20 before the
//      frame cannot leak in), or M[hi] (min / max of frames that start at the partition's first row); first / last values and
//      lag / lead are gathers.
// Frames: ROWS with any bounds; RANGE with UNBOUNDED / CURRENT ROW bounds (the default frames) and with value offsets over one
// numeric / date ORDER BY key (per-row binary searches in the sorted partition); min / max need a frame that starts at UNBOUNDED
// PRECEDING.
#include <memory>
#include <type_traits>
#include <vector>
#include "common.cuh"
#include "primitives.cuh"
#include "sort.cuh"
#include "strings.cuh"

namespace sb {

constexpr int WIN_THREADS = 256;
constexpr int WIN_ITEMS = 8;
constexpr int WIN_TILE = WIN_THREADS * WIN_ITEMS;

static inline unsigned wblocks(int64_t n, int per = 256) { return (unsigned)((n + per - 1) / per); }

// ---- adjacent-row comparison -------------------------------------------------------------------------------------------
struct CmpCols {
  int n;
  const void *data[8];
  const uint8_t *valid[8];
  int32_t type[8];
};
__device__ __forceinline__ bool cell_differs(const CmpCols &c, int k, int64_t a, int64_t b) {
  const bool va = bit_valid(c.valid[k], a), vb = bit_valid(c.valid[k], b);
  if (va != vb) return true;
  if (!va) return false;
  switch (c.type[k]) {
    case SB_FLOAT64: {
      const double x = ((const double *)c.data[k])[a], y = ((const double *)c.data[k])[b];
      return (x == 0.0 ? 0ll : double_bits_canonical(x)) != (y == 0.0 ? 0ll : double_bits_canonical(y));
    }
    case SB_FLOAT32: {
      const float x = ((const float *)c.data[k])[a], y = ((const float *)c.data[k])[b];
      return (x == 0.0f ? 0 : float_bits_canonical(x)) != (y == 0.0f ? 0 : float_bits_canonical(y));
    }
    default: return load_i64(c.data[k], c.type[k], a) != load_i64(c.data[k], c.type[k], b);
  }
}
// seg[i] = 1 when row i starts a partition, peer[i] = 1 when it starts a peer group (npart columns first, then the order columns)
__global__ void heads_kernel(CmpCols c, int npart, int64_t n, int32_t *__restrict__ seg, int32_t *__restrict__ peer) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool s = i == 0, p = i == 0;
  if (i > 0) {
    for (int k = 0; k < c.n && !s; k++) {
      const bool d = cell_differs(c, k, i - 1, i);
      if (d && k < npart) s = true;
      if (d) p = true;
    }
  }
  seg[i] = s;
  peer[i] = s || p;
}
// ids (dense, 0-based) from the exclusive prefix of the head flags; first[id] = row of the head
__global__ void ids_kernel(const int32_t *__restrict__ head, const int32_t *__restrict__ excl, int64_t n, int32_t *__restrict__ id,
                           int64_t *__restrict__ first) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t g = excl[i] + head[i] - 1;
  id[i] = g;
  if (head[i]) first[g] = i;
}

// ---- segmented inclusive scan (restarts where head != 0) -------------------------------------------------------------------
enum { SEG_SUM = 0, SEG_MIN = 1, SEG_MAX = 2 };
template <typename T> struct SegElem { T v; int has; int head; };

template <typename T, int OP> __device__ __forceinline__ T seg_op(T a, T b) {
  if (OP == SEG_SUM) return a + b;
  if (OP == SEG_MIN) return b < a ? b : a;
  return b > a ? b : a;
}
// doubles order like SQLOrderingUtil.compareDoubles: NaN is larger than everything
template <> __device__ __forceinline__ double seg_op<double, SEG_MIN>(double a, double b) { return (b < a || a != a) ? b : a; }
template <> __device__ __forceinline__ double seg_op<double, SEG_MAX>(double a, double b) { return (b > a || b != b) ? b : a; }

template <typename T, int OP> __device__ __forceinline__ SegElem<T> seg_combine(const SegElem<T> &a, const SegElem<T> &b) {   // a before b
  if (b.head) return b;
  SegElem<T> r;
  r.head = a.head;
  r.has = a.has | b.has;
  r.v = (a.has && b.has) ? seg_op<T, OP>(a.v, b.v) : (a.has ? a.v : b.v);
  return r;
}

// PHASE 0: tile aggregates only.  PHASE 1: outputs, starting from carry[tile] (the inclusive result just before the tile).
template <typename T, int OP, int PHASE>
__global__ void __launch_bounds__(WIN_THREADS) seg_scan_kernel(const T *__restrict__ v, const uint8_t *__restrict__ has, const int32_t *__restrict__ head,
                                                               int64_t n, T *__restrict__ agg_v, uint8_t *__restrict__ agg_has,
                                                               int32_t *__restrict__ agg_head, const T *__restrict__ carry_v,
                                                               const uint8_t *__restrict__ carry_has, T *__restrict__ out_v,
                                                               uint8_t *__restrict__ out_has) {
  __shared__ T sh_v[WIN_THREADS];
  __shared__ int sh_has[WIN_THREADS], sh_head[WIN_THREADS];
  const int tid = threadIdx.x;
  const int64_t base = (int64_t)blockIdx.x * WIN_TILE + (int64_t)tid * WIN_ITEMS;
  SegElem<T> e[WIN_ITEMS];
  SegElem<T> run;
  run.v = 0; run.has = 0; run.head = 0;
#pragma unroll
  for (int k = 0; k < WIN_ITEMS; k++) {
    const int64_t i = base + k;
    SegElem<T> x;
    x.v = 0; x.has = 0; x.head = 0;
    if (i < n) {
      x.has = has ? has[i] != 0 : 1;
      x.v = x.has ? v[i] : (T)0;
      x.head = head[i] != 0;
    }
    run = k == 0 ? x : seg_combine<T, OP>(run, x);
    e[k] = run;
  }
  sh_v[tid] = run.v; sh_has[tid] = run.has; sh_head[tid] = run.head;
  __syncthreads();
  for (int d = 1; d < WIN_THREADS; d <<= 1) {   // inclusive scan of the thread aggregates
    SegElem<T> a, b;
    const bool take = tid >= d;
    if (take) {
      a.v = sh_v[tid - d]; a.has = sh_has[tid - d]; a.head = sh_head[tid - d];
      b.v = sh_v[tid]; b.has = sh_has[tid]; b.head = sh_head[tid];
      b = seg_combine<T, OP>(a, b);
    }
    __syncthreads();
    if (take) { sh_v[tid] = b.v; sh_has[tid] = b.has; sh_head[tid] = b.head; }
    __syncthreads();
  }
  if (PHASE == 0) {
    if (tid == WIN_THREADS - 1) {
      agg_v[blockIdx.x] = sh_v[tid];
      agg_has[blockIdx.x] = (uint8_t)sh_has[tid];
      agg_head[blockIdx.x] = sh_head[tid];
    }
    return;
  }
  SegElem<T> before;   // everything before this thread's items: carry, then the preceding threads of the tile
  before.v = 0; before.has = 0; before.head = 0;
  if (blockIdx.x > 0) { before.v = carry_v[blockIdx.x]; before.has = carry_has[blockIdx.x]; }
  if (tid > 0) {
    SegElem<T> p;
    p.v = sh_v[tid - 1]; p.has = sh_has[tid - 1]; p.head = sh_head[tid - 1];
    before = seg_combine<T, OP>(before, p);
  }
#pragma unroll
  for (int k = 0; k < WIN_ITEMS; k++) {
    const int64_t i = base + k;
    if (i >= n) break;
    const SegElem<T> r = seg_combine<T, OP>(before, e[k]);
    out_v[i] = r.v;
    out_has[i] = (uint8_t)r.has;
  }
}
__global__ void shift_carry_kernel_u8(const uint8_t *in, int64_t n, uint8_t *out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i == 0 ? 0 : in[i - 1];
}
template <typename T> __global__ void shift_carry_kernel(const T *in, int64_t n, T *out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i == 0 ? (T)0 : in[i - 1];
}

template <typename T, int OP>
static void seg_scan(const T *v, const uint8_t *has, const int32_t *head, int64_t n, T *out_v, uint8_t *out_has, cudaStream_t st) {
  if (n == 0) return;
  const int64_t tiles = (n + WIN_TILE - 1) / WIN_TILE;
  if (tiles == 1) {
    seg_scan_kernel<T, OP, 1><<<1, WIN_THREADS, 0, st>>>(v, has, head, n, nullptr, nullptr, nullptr, nullptr, nullptr, out_v, out_has);
    SB_LAUNCH_CHECK();
    return;
  }
  Scratch agg_v(tiles * sizeof(T) + 16, st), agg_has(tiles + 16, st), agg_head(tiles * 4 + 16, st);
  Scratch inc_v(tiles * sizeof(T) + 16, st), inc_has(tiles + 16, st), car_v(tiles * sizeof(T) + 16, st), car_has(tiles + 16, st);
  seg_scan_kernel<T, OP, 0><<<(unsigned)tiles, WIN_THREADS, 0, st>>>(v, has, head, n, agg_v.as<T>(), agg_has.as<uint8_t>(), agg_head.as<int32_t>(),
                                                                     nullptr, nullptr, nullptr, nullptr);
  SB_LAUNCH_CHECK();
  seg_scan<T, OP>(agg_v.as<T>(), agg_has.as<uint8_t>(), agg_head.as<int32_t>(), tiles, inc_v.as<T>(), inc_has.as<uint8_t>(), st);
  shift_carry_kernel<T><<<wblocks(tiles), 256, 0, st>>>(inc_v.as<T>(), tiles, car_v.as<T>());
  shift_carry_kernel_u8<<<wblocks(tiles), 256, 0, st>>>(inc_has.as<uint8_t>(), tiles, car_has.as<uint8_t>());
  SB_LAUNCH_CHECK();
  seg_scan_kernel<T, OP, 1><<<(unsigned)tiles, WIN_THREADS, 0, st>>>(v, has, head, n, nullptr, nullptr, nullptr, car_v.as<T>(), car_has.as<uint8_t>(),
                                                                     out_v, out_has);
  SB_LAUNCH_CHECK();
}

// ---- per-row bounds ---------------------------------------------------------------------------------------------------------
struct Bounds {
  const int32_t *seg_id, *peer_id;
  const int64_t *seg_first, *peer_first;
  int64_t nseg, npeer, n;
  // the single ORDER BY key, for RANGE frames with value offsets
  const void *okey;
  const uint8_t *okey_valid;
  int32_t okey_type, asc, nulls_first;
};
__device__ __forceinline__ int64_t seg_start_of(const Bounds &b, int64_t i) { return b.seg_first[b.seg_id[i]]; }
__device__ __forceinline__ int64_t seg_end_of(const Bounds &b, int64_t i) {
  const int32_t g = b.seg_id[i];
  return g + 1 < b.nseg ? b.seg_first[g + 1] : b.n;
}
__device__ __forceinline__ int64_t peer_start_of(const Bounds &b, int64_t i) { return b.peer_first[b.peer_id[i]]; }
__device__ __forceinline__ int64_t peer_end_of(const Bounds &b, int64_t i) {
  const int32_t g = b.peer_id[i];
  return g + 1 < b.npeer ? b.peer_first[g + 1] : b.n;
}
// Where does row j's order key sort relative to `bound` in the partition's order: -1 before, 0 equal, +1 after.  NULL keys sit
// where the null ordering put them.  F64: keys and bounds are doubles (SQLOrderingUtil.compareDoubles: NaN largest).
template <bool F64>
__device__ __forceinline__ int key_vs(const Bounds &b, int64_t j, int64_t bound_i, double bound_d) {
  if (!bit_valid(b.okey_valid, j)) return b.nulls_first ? -1 : 1;
  int c;
  if (F64) {
    const double v = b.okey_type == SB_FLOAT32 ? (double)((const float *)b.okey)[j] : ((const double *)b.okey)[j];
    const bool vn = v != v, bn = bound_d != bound_d;
    c = v == bound_d ? 0 : (vn || bn) ? (int)vn - (int)bn : (v < bound_d ? -1 : 1);
  } else {
    const int64_t v = load_i64(b.okey, b.okey_type, j);
    c = v == bound_i ? 0 : (v < bound_i ? -1 : 1);
  }
  return b.asc ? c : -c;
}
// first row of [s, e] whose key does not sort before the bound (AFTER = false) / first row whose key sorts after it (AFTER = true)
template <bool F64, bool AFTER>
__device__ __forceinline__ int64_t range_search(const Bounds &b, int64_t s, int64_t e, int64_t bound_i, double bound_d) {
  int64_t lo = s, hi = e + 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const int c = key_vs<F64>(b, mid, bound_i, bound_d);
    if (AFTER ? c <= 0 : c < 0) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ int64_t sat_add(int64_t a, int64_t x) {
  const int64_t r = (int64_t)((uint64_t)a + (uint64_t)x);
  if (x > 0 && r < a) return INT64_MAX;
  if (x < 0 && r > a) return INT64_MIN;
  return r;
}
// frame of row i as [lo, hi] (empty when lo > hi)
__device__ __forceinline__ void frame_of(const Bounds &b, int64_t i, int frame_type, int64_t lower, int64_t upper, int64_t &lo, int64_t &hi) {
  const int64_t s = seg_start_of(b, i), e = seg_end_of(b, i) - 1;
  if (frame_type != SB_FRAME_ROWS) {
    // RANGE: UNBOUNDED -> the partition's end, CURRENT ROW (0) -> the peer group's end, otherwise a VALUE offset: the bound is the
    // row's key plus the offset in the direction of the ordering (WindowEvaluatorFactoryBase.createBoundOrdering: Add for ASC,
    // Subtract for DESC) and the frame holds the rows whose keys lie between the two bounds; a NULL key has only its peers
    const bool f64 = frame_type == SB_FRAME_RANGE_F64;
    const bool null_key = b.okey && !bit_valid(b.okey_valid, i);
    int64_t vi = 0;
    double vd = 0.0;
    if (b.okey && !null_key) {
      if (f64) vd = b.okey_type == SB_FLOAT32 ? (double)((const float *)b.okey)[i] : ((const double *)b.okey)[i];
      else vi = load_i64(b.okey, b.okey_type, i);
    }
    if (lower == SB_UNBOUNDED_PRECEDING) lo = s;
    else if (lower == 0 || null_key || !b.okey) lo = peer_start_of(b, i);
    else if (f64) {
      const double off = __longlong_as_double(lower);
      lo = range_search<true, false>(b, s, e, 0, b.asc ? vd + off : vd - off);
    } else lo = range_search<false, false>(b, s, e, b.asc ? sat_add(vi, lower) : sat_add(vi, -lower), 0.0);
    if (upper == SB_UNBOUNDED_FOLLOWING) hi = e;
    else if (upper == 0 || null_key || !b.okey) hi = peer_end_of(b, i) - 1;
    else if (f64) {
      const double off = __longlong_as_double(upper);
      hi = range_search<true, true>(b, s, e, 0, b.asc ? vd + off : vd - off) - 1;
    } else hi = range_search<false, true>(b, s, e, b.asc ? sat_add(vi, upper) : sat_add(vi, -upper), 0.0) - 1;
    return;
  }
  lo = lower == SB_UNBOUNDED_PRECEDING ? s : i + lower;
  hi = upper == SB_UNBOUNDED_FOLLOWING ? e : i + upper;
  if (lo < s) lo = s;
  if (hi > e) hi = e;
}

// ---- the functions ------------------------------------------------------------------------------------------------------------
__global__ void rank_kernel(Bounds b, int func, int64_t param, int32_t *__restrict__ out_i32, double *__restrict__ out_f64) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b.n) return;
  const int64_t s = seg_start_of(b, i), e = seg_end_of(b, i), size = e - s;
  const int64_t row_number = i - s + 1, rank = peer_start_of(b, i) - s + 1;
  switch (func) {
    case SB_WIN_ROW_NUMBER: out_i32[i] = (int32_t)row_number; break;
    case SB_WIN_RANK: out_i32[i] = (int32_t)rank; break;
    case SB_WIN_DENSE_RANK: out_i32[i] = b.peer_id[i] - b.peer_id[s] + 1; break;
    case SB_WIN_PERCENT_RANK: out_f64[i] = size > 1 ? (double)(rank - 1) / (double)(size - 1) : 0.0; break;   // windowExpressions.scala PercentRank
    case SB_WIN_CUME_DIST: out_f64[i] = (double)(peer_end_of(b, i) - s) / (double)size; break;
    default: {   // NTILE (windowExpressions.scala NTile: the first size % n buckets hold one row more)
      const int64_t bs = size / param, rem = size % param, r = row_number - 1;
      out_i32[i] = (int32_t)(r < (bs + 1) * rem ? r / (bs + 1) + 1 : rem + (r - (bs + 1) * rem) / (bs > 0 ? bs : 1) + 1);
    }
  }
}
// gather index of lag / lead / first_value / last_value (-1 = NULL)
__global__ void pick_kernel(Bounds b, int func, int frame_type, int64_t lower, int64_t upper, int64_t param, int64_t *__restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b.n) return;
  int64_t j = -1;
  if (func == SB_WIN_LAG || func == SB_WIN_LEAD) {
    j = func == SB_WIN_LAG ? i - param : i + param;
    if (j < seg_start_of(b, i) || j >= seg_end_of(b, i)) j = -1;
  } else {
    int64_t lo, hi;
    frame_of(b, i, frame_type, lower, upper, lo, hi);
    if (lo <= hi) j = func == SB_WIN_FIRST_VALUE ? lo : hi;
  }
  idx[i] = j;
}
// Block sums of the widened double inputs (NULL = 0.0): level j holds the sums of the aligned 2^j-row blocks, level 0 is the
// input itself.  A double frame that does not start at its partition's first row is summed from the blocks that lie inside it,
// so inf / NaN / large values outside the frame cannot reach its result (a difference of running sums would let them).
constexpr int WIN_MAX_LEVELS = 32;
struct BlockSums {
  const double *level[WIN_MAX_LEVELS];
};
__global__ void block_sum_level_kernel(const double *__restrict__ below, int64_t m, double *__restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) out[k] = below[2 * k] + below[2 * k + 1];
}
// +0.0 (Spark's sums start from zero: Sum.scala coalesce(sum, 0) + x) plus, left to right, the largest aligned blocks that tile
// [lo, hi]: at most 2 log2(hi - lo + 1) of them
__device__ __forceinline__ double frame_block_sum(const BlockSums &bs, int64_t lo, int64_t hi) {
  double acc = 0.0;
  while (lo <= hi) {
    int j = 63 - __clzll((unsigned long long)(hi - lo + 1));   // the widest block that fits ...
    if (lo != 0 && __ffsll(lo) - 1 < j) j = __ffsll(lo) - 1;   // ... and is aligned at lo
    acc = acc + bs.level[j][lo >> j];
    lo += 1ll << j;
  }
  return acc;
}

// sum / count / avg over the frame.  C = running count; S = running sum of the non-NULL inputs.  Integers take S[hi] - S[lo - 1]
// (exact modulo 2^64, like Spark's wrapping long sum).  Doubles take +0.0 + S[hi] when the frame starts at the partition's first
// row and the block sums (bs) otherwise.
template <typename T>
__global__ void frame_sum_kernel(Bounds b, int func, int frame_type, int64_t lower, int64_t upper, const T *__restrict__ S, const int64_t *__restrict__ C,
                                 BlockSums bs, void *__restrict__ out, uint32_t *__restrict__ out_valid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < b.n;
  bool valid = false;
  if (in) {
    int64_t lo, hi;
    frame_of(b, i, frame_type, lower, upper, lo, hi);
    T sum = 0;
    int64_t cnt = 0;
    if (lo <= hi) {
      const int64_t s = seg_start_of(b, i);
      sum = S ? S[hi] : (T)0;
      cnt = C[hi];
      if (lo > s) {
        if (S) {
          if constexpr (std::is_same<T, double>::value) sum = frame_block_sum(bs, lo, hi);
          else sum -= S[lo - 1];
        }
        cnt -= C[lo - 1];
      } else if constexpr (std::is_same<T, double>::value) {
        sum = sum + 0.0;   // a lone -0.0 sums to +0.0
      }
    }
    if (func == SB_WIN_COUNT) {
      ((int64_t *)out)[i] = cnt;
      valid = true;
    } else if (func == SB_WIN_SUM) {
      ((T *)out)[i] = sum;
      valid = cnt > 0;
    } else {   // AVG: double sum / count (Average.scala:80)
      ((double *)out)[i] = cnt > 0 ? (double)sum / (double)cnt : 0.0;
      valid = cnt > 0;
    }
  }
  if (out_valid) {
    const uint32_t w = __ballot_sync(0xffffffffu, in && valid);
    if ((threadIdx.x & 31) == 0 && i - (i & 31) < b.n) out_valid[i >> 5] = w;
  }
}
// min / max of a frame that starts at the partition's first row: the running value at the frame's last row
__global__ void frame_pick_last_kernel(Bounds b, int frame_type, int64_t lower, int64_t upper, int64_t *__restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b.n) return;
  int64_t lo, hi;
  frame_of(b, i, frame_type, lower, upper, lo, hi);
  idx[i] = lo <= hi ? hi : -1;
}

// input column widened to int64 / double for the scans; has[i] = not NULL
__global__ void widen_kernel(const void *__restrict__ data, const uint8_t *__restrict__ valid, int32_t type, int64_t n, int64_t *__restrict__ vi,
                             double *__restrict__ vd, uint8_t *__restrict__ has, int64_t *__restrict__ ones) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool ok = bit_valid(valid, i);
  has[i] = ok;
  if (ones) ones[i] = ok ? 1 : 0;
  if (vd) vd[i] = !ok ? 0.0 : type == SB_FLOAT64 ? ((const double *)data)[i] : type == SB_FLOAT32 ? (double)((const float *)data)[i] : (double)load_i64(data, type, i);
  if (vi) vi[i] = ok ? load_i64(data, type, i) : 0;
}
template <typename T>
__global__ void narrow_kernel(const T *__restrict__ v, const uint8_t *__restrict__ has, const int64_t *__restrict__ idx, int32_t type, int64_t n, void *__restrict__ out,
                              uint32_t *__restrict__ out_valid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < n;
  bool valid = false;
  if (in) {
    const int64_t j = idx[i];
    valid = j >= 0 && has[j];
    const T x = valid ? v[j] : (T)0;
    switch (type) {
      case SB_BOOL: case SB_INT8: ((int8_t *)out)[i] = (int8_t)x; break;
      case SB_INT16: ((int16_t *)out)[i] = (int16_t)x; break;
      case SB_INT32: case SB_DATE32: ((int32_t *)out)[i] = (int32_t)x; break;
      case SB_FLOAT32: ((float *)out)[i] = (float)x; break;
      case SB_FLOAT64: ((double *)out)[i] = (double)x; break;
      default: ((int64_t *)out)[i] = (int64_t)x; break;
    }
  }
  const uint32_t w = __ballot_sync(0xffffffffu, in && valid);
  if ((threadIdx.x & 31) == 0 && i - (i & 31) < n) out_valid[i >> 5] = w;
}
__global__ void u32_to_i64_kernel_w(const uint32_t *__restrict__ in, int64_t n, int64_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i];
}

static bool is_float(int32_t t) { return t == SB_FLOAT32 || t == SB_FLOAT64; }

}  // namespace sb

using namespace sb;

extern "C" int sb_window(const sb_table *in, const int32_t *partition_cols, int32_t npart, const sb_sort_order *orders, int32_t norders,
                         const sb_window_spec *specs, int32_t nspecs, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(in && out && npart >= 0 && norders >= 0 && nspecs >= 0, "bad argument");
  SB_REQUIRE(npart + norders <= 8, "at most 8 partition + order columns");
  SB_REQUIRE((npart == 0 || partition_cols) && (norders == 0 || orders) && (nspecs == 0 || specs), "null argument");
  cudaStream_t st = stream_of(s);
  const int64_t n = in->nrows;
  SB_REQUIRE(n < (1ll << 31), "sb_window takes fewer than 2^31 rows per call");
  const int ncols_in = (int)in->cols.size();
  for (int k = 0; k < npart; k++) SB_REQUIRE(partition_cols[k] >= 0 && partition_cols[k] < ncols_in, "partition column %d out of range", partition_cols[k]);
  for (int k = 0; k < norders; k++) SB_REQUIRE(orders[k].col >= 0 && orders[k].col < ncols_in, "order column %d out of range", orders[k].col);

  // 1. sort by (partition keys ASC NULLS FIRST, order spec)
  std::vector<sb_sort_order> so;
  for (int k = 0; k < npart; k++) so.push_back(sb_sort_order{partition_cols[k], 1, 1, 0});
  for (int k = 0; k < norders; k++) so.push_back(orders[k]);
  sb_table *sorted = nullptr;
  if (!so.empty() && n > 0) {
    Scratch perm(n * 4 + 16, st), perm64(n * 8 + 16, st);
    sort_permutation_impl(in, so.data(), (int32_t)so.size(), perm.as<uint32_t>(), st);
    u32_to_i64_kernel_w<<<wblocks(n), 256, 0, st>>>(perm.as<uint32_t>(), n, perm64.as<int64_t>());
    SB_LAUNCH_CHECK();
    sorted = gather_table(in, perm64.as<int64_t>(), n, false, st);
  } else {
    sorted = table_new(n);
    for (auto &c : in->cols) sorted->cols.push_back(column_share(c));
  }
  struct Guard { sb_table *t; ~Guard() { if (t) table_free(t); } } guard{sorted};

  // 2. heads (string key columns compare through their dictionary codes)
  EncodedView ev;
  {
    std::vector<int> scols;
    for (auto &o : so)
      if (sorted->cols[o.col].type == SB_STRING) scols.push_back(o.col);
    if (!scols.empty()) encode_string_columns(sorted, scols, nullptr, st, ev);
  }
  const sb_table *keys = ev.view ? ev.view : sorted;
  CmpCols cc;
  cc.n = (int)so.size();
  for (int k = 0; k < cc.n; k++) {
    const Column &c = keys->cols[so[k].col];
    cc.data[k] = c.d();
    cc.valid[k] = c.v();
    cc.type[k] = c.type;
  }
  Scratch seg_head(n * 4 + 16, st), peer_head(n * 4 + 16, st), excl(n * 4 + 16, st), seg_id(n * 4 + 16, st), peer_id(n * 4 + 16, st), totals(16, st);
  Scratch seg_first(n * 8 + 16, st), peer_first(n * 8 + 16, st);
  int32_t counts[2] = {0, 0};
  if (n > 0) {
    heads_kernel<<<wblocks(n), 256, 0, st>>>(cc, npart, n, seg_head.as<int32_t>(), peer_head.as<int32_t>());
    SB_LAUNCH_CHECK();
    exclusive_scan_i32(seg_head.as<int32_t>(), excl.as<int32_t>(), n, totals.as<int32_t>(), st);
    ids_kernel<<<wblocks(n), 256, 0, st>>>(seg_head.as<int32_t>(), excl.as<int32_t>(), n, seg_id.as<int32_t>(), seg_first.as<int64_t>());
    SB_LAUNCH_CHECK();
    exclusive_scan_i32(peer_head.as<int32_t>(), excl.as<int32_t>(), n, totals.as<int32_t>() + 1, st);
    ids_kernel<<<wblocks(n), 256, 0, st>>>(peer_head.as<int32_t>(), excl.as<int32_t>(), n, peer_id.as<int32_t>(), peer_first.as<int64_t>());
    SB_LAUNCH_CHECK();
    SB_CUDA(cudaMemcpyAsync(counts, totals.ptr, 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  Bounds b{seg_id.as<int32_t>(), peer_id.as<int32_t>(), seg_first.as<int64_t>(), peer_first.as<int64_t>(), counts[0], counts[1], n,
           nullptr, nullptr, 0, 1, 1};
  if (norders == 1) {   // value-offset RANGE frames read the (single) order key
    const Column &ok = sorted->cols[orders[0].col];
    if (ok.type != SB_STRING && ok.type != SB_DECIMAL64 && ok.type != SB_DECIMAL128 && ok.type != SB_BOOL) {
      b.okey = ok.d();
      b.okey_valid = ok.v();
      b.okey_type = ok.type;
      b.asc = orders[0].ascending != 0;
      b.nulls_first = orders[0].nulls_first != 0;
    }
  }

  // 3. output = sorted input ++ one column per window expression
  sb_table *t = table_new(n);
  try {
    for (auto &c : sorted->cols) t->cols.push_back(column_share(c));
    for (int k = 0; k < nspecs; k++) {
      const sb_window_spec &w = specs[k];
      const bool ranking = w.func >= SB_WIN_ROW_NUMBER && w.func <= SB_WIN_NTILE;
      if (ranking) {
        if (w.func == SB_WIN_NTILE) SB_REQUIRE(w.param > 0, "ntile needs a positive bucket count");
        const bool f64 = w.func == SB_WIN_PERCENT_RANK || w.func == SB_WIN_CUME_DIST;
        Column c = column_alloc(f64 ? SB_FLOAT64 : SB_INT32, 0, n, false, st);
        t->cols.push_back(c);
        if (n > 0) {
          rank_kernel<<<wblocks(n), 256, 0, st>>>(b, w.func, w.param, f64 ? nullptr : (int32_t *)c.data->ptr, f64 ? (double *)c.data->ptr : nullptr);
          SB_LAUNCH_CHECK();
        }
        continue;
      }
      SB_REQUIRE(w.func >= SB_WIN_LAG && w.func <= SB_WIN_LAST_VALUE, "unknown window function %d", w.func);
      SB_REQUIRE(w.col >= 0 && w.col < ncols_in, "window function input column %d out of range", w.col);
      SB_REQUIRE(w.frame_type == SB_FRAME_ROWS || w.frame_type == SB_FRAME_RANGE || w.frame_type == SB_FRAME_RANGE_F64, "unknown frame type %d",
                 w.frame_type);
      if (w.frame_type != SB_FRAME_ROWS && w.func != SB_WIN_LAG && w.func != SB_WIN_LEAD) {
        const bool offsets = (w.lower != SB_UNBOUNDED_PRECEDING && w.lower != 0) || (w.upper != SB_UNBOUNDED_FOLLOWING && w.upper != 0);
        if (offsets) {   // SpecifiedWindowFrame with value bounds: exactly one numeric ORDER BY expression (windowExpressions.scala checkInputDataTypes)
          if (!b.okey) fail(SB_ERR_UNSUPPORTED, "a RANGE frame with value offsets needs exactly one numeric / date ORDER BY column");
          const bool fkey = b.okey_type == SB_FLOAT32 || b.okey_type == SB_FLOAT64;
          SB_REQUIRE(fkey == (w.frame_type == SB_FRAME_RANGE_F64), "RANGE offsets are doubles (SB_FRAME_RANGE_F64) exactly when the ORDER BY column is floating point");
        }
      }
      const Column &src = sorted->cols[w.col];
      if (w.func == SB_WIN_LAG || w.func == SB_WIN_LEAD || w.func == SB_WIN_FIRST_VALUE || w.func == SB_WIN_LAST_VALUE) {
        if (w.func == SB_WIN_LAG || w.func == SB_WIN_LEAD) SB_REQUIRE(w.param >= 0, "lag / lead offset must not be negative");
        Scratch idx(n * 8 + 16, st);
        if (n > 0) {
          pick_kernel<<<wblocks(n), 256, 0, st>>>(b, w.func, w.frame_type, w.lower, w.upper, w.param, idx.as<int64_t>());
          SB_LAUNCH_CHECK();
        }
        t->cols.push_back(gather_column(src, idx.as<int64_t>(), n, true, st));
        continue;
      }
      if (src.type == SB_STRING || src.type == SB_DECIMAL64) fail(SB_ERR_UNSUPPORTED, "window aggregates over string / decimal columns are not implemented");
      const bool fl = is_float(src.type);
      Scratch vi(fl ? 0 : n * 8 + 16, st), vd(fl ? n * 8 + 16 : 0, st), has(n + 16, st), ones(n * 8 + 16, st);
      if (n > 0) {
        widen_kernel<<<wblocks(n), 256, 0, st>>>(src.d(), src.v(), src.type, n, fl ? nullptr : vi.as<int64_t>(), fl ? vd.as<double>() : nullptr,
                                                has.as<uint8_t>(), ones.as<int64_t>());
        SB_LAUNCH_CHECK();
      }
      if (w.func == SB_WIN_MIN || w.func == SB_WIN_MAX) {
        if (w.lower != SB_UNBOUNDED_PRECEDING) fail(SB_ERR_UNSUPPORTED, "min / max over a frame that does not start at UNBOUNDED PRECEDING is not implemented");
        Scratch run(n * 8 + 16, st), run_has(n + 16, st), idx(n * 8 + 16, st);
        Column c = column_alloc(src.type, src.scale, n, true, st);
        t->cols.push_back(c);
        if (n > 0) {
          if (fl) {
            if (w.func == SB_WIN_MIN) seg_scan<double, SEG_MIN>(vd.as<double>(), has.as<uint8_t>(), seg_head.as<int32_t>(), n, run.as<double>(), run_has.as<uint8_t>(), st);
            else seg_scan<double, SEG_MAX>(vd.as<double>(), has.as<uint8_t>(), seg_head.as<int32_t>(), n, run.as<double>(), run_has.as<uint8_t>(), st);
          } else {
            if (w.func == SB_WIN_MIN) seg_scan<int64_t, SEG_MIN>(vi.as<int64_t>(), has.as<uint8_t>(), seg_head.as<int32_t>(), n, run.as<int64_t>(), run_has.as<uint8_t>(), st);
            else seg_scan<int64_t, SEG_MAX>(vi.as<int64_t>(), has.as<uint8_t>(), seg_head.as<int32_t>(), n, run.as<int64_t>(), run_has.as<uint8_t>(), st);
          }
          frame_pick_last_kernel<<<wblocks(n), 256, 0, st>>>(b, w.frame_type, w.lower, w.upper, idx.as<int64_t>());
          SB_LAUNCH_CHECK();
          if (fl) narrow_kernel<double><<<wblocks(n), 256, 0, st>>>(run.as<double>(), run_has.as<uint8_t>(), idx.as<int64_t>(), src.type, n, c.data->ptr, (uint32_t *)c.validity->ptr);
          else narrow_kernel<int64_t><<<wblocks(n), 256, 0, st>>>(run.as<int64_t>(), run_has.as<uint8_t>(), idx.as<int64_t>(), src.type, n, c.data->ptr, (uint32_t *)c.validity->ptr);
          SB_LAUNCH_CHECK();
        }
        continue;
      }
      // SUM / COUNT / AVG: running sum and running count, then frame differences
      SB_REQUIRE(w.func == SB_WIN_SUM || w.func == SB_WIN_COUNT || w.func == SB_WIN_AVG, "unknown window function %d", w.func);
      const bool sum_f64 = fl || w.func == SB_WIN_AVG;   // Average sums as double (Average.scala:80)
      Scratch S(n * 8 + 16, st), S_has(n + 16, st), Cn(n * 8 + 16, st), C_has(n + 16, st), vavg(!fl && w.func == SB_WIN_AVG ? n * 8 + 16 : 0, st);
      const int32_t out_type = w.func == SB_WIN_COUNT ? SB_INT64 : (sum_f64 ? SB_FLOAT64 : SB_INT64);
      Column c = column_alloc(out_type, 0, n, w.func != SB_WIN_COUNT, st);
      t->cols.push_back(c);
      if (n > 0) {
        seg_scan<int64_t, SEG_SUM>(ones.as<int64_t>(), nullptr, seg_head.as<int32_t>(), n, Cn.as<int64_t>(), C_has.as<uint8_t>(), st);
        if (w.func != SB_WIN_COUNT) {
          if (sum_f64) {
            double *vals = vd.as<double>();
            if (!fl) {   // integral input of an average: widen to double first
              widen_kernel<<<wblocks(n), 256, 0, st>>>(src.d(), src.v(), src.type, n, nullptr, vavg.as<double>(), has.as<uint8_t>(), nullptr);
              SB_LAUNCH_CHECK();
              vals = vavg.as<double>();
            }
            seg_scan<double, SEG_SUM>(vals, has.as<uint8_t>(), seg_head.as<int32_t>(), n, S.as<double>(), S_has.as<uint8_t>(), st);
            // block sums for frames that may start after the partition's first row (about n more doubles)
            BlockSums bs{};
            bs.level[0] = vals;
            Scratch blocks(w.lower != SB_UNBOUNDED_PRECEDING ? n * 8 + 16 : 0, st);
            if (w.lower != SB_UNBOUNDED_PRECEDING) {
              double *next = blocks.as<double>();
              for (int j = 1; (n >> j) > 0; j++) {
                const int64_t m = n >> j;
                block_sum_level_kernel<<<wblocks(m), 256, 0, st>>>(bs.level[j - 1], m, next);
                SB_LAUNCH_CHECK();
                bs.level[j] = next;
                next += m;
              }
            }
            frame_sum_kernel<double><<<wblocks(n), 256, 0, st>>>(b, w.func, w.frame_type, w.lower, w.upper, S.as<double>(), Cn.as<int64_t>(), bs,
                                                                 c.data->ptr, c.validity ? (uint32_t *)c.validity->ptr : nullptr);
          } else {
            seg_scan<int64_t, SEG_SUM>(vi.as<int64_t>(), has.as<uint8_t>(), seg_head.as<int32_t>(), n, S.as<int64_t>(), S_has.as<uint8_t>(), st);
            frame_sum_kernel<int64_t><<<wblocks(n), 256, 0, st>>>(b, w.func, w.frame_type, w.lower, w.upper, S.as<int64_t>(), Cn.as<int64_t>(), BlockSums{},
                                                                  c.data->ptr, c.validity ? (uint32_t *)c.validity->ptr : nullptr);
          }
        } else {
          frame_sum_kernel<int64_t><<<wblocks(n), 256, 0, st>>>(b, w.func, w.frame_type, w.lower, w.upper, nullptr, Cn.as<int64_t>(), BlockSums{},
                                                                c.data->ptr, nullptr);
        }
        SB_LAUNCH_CHECK();
      }
    }
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
  SB_CUDA(cudaStreamSynchronize(st));   // the scratch buffers above die with this frame
  SB_API_END
}
