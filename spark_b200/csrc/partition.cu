// partition.cu -- ShuffleExchangeExec map side on the GPU.
//
// Reference path replaced (citations relative to the reference tree):
//   partition id  = Pmod(Murmur3Hash(keys, 42), n)      sql/catalyst/.../plans/physical/partitioning.scala:339-341
//   Murmur3       = common/unsafe/.../hash/Murmur3_x86_32.java:47-150, type dispatch hash.scala:707-760
//   grouping rows by partition id = UnsafeShuffleWriter + ShuffleInMemorySorter radix on the partition
//                   bytes of PackedRecordPointer (core/src/main/java/org/apache/spark/shuffle/sort/
//                   ShuffleInMemorySorter.java:202-225) / BypassMergeSortShuffleWriter for n <= 200.
//
// GPU design (HBM-bound integer work, no tensor cores): a stable single-pass multisplit.
//   K1 pid_hist   : one coalesced read of the key columns, Murmur3 chain in registers, pid stored as
//                   int32, per-block shared-memory histogram -> hist[p][block]
//   K2 scan       : exclusive scan over hist in (partition, block) order -> every block's first output
//                   slot for every partition, and the partition boundaries
//   K3 scatter    : each block re-walks its contiguous chunk; every warp owns a contiguous sub-chunk and
//                   keeps running per-partition cursors in shared memory; ranks inside a 32-row group come
//                   from __match_any_sync, so arrival order inside a partition is preserved (stable);
//                   all fixed-width payload columns are moved with one coalesced read and one write each.
// Algorithmic bytes: 2 x rowbytes per row (SURVEY.md 8d); overhead: keys re-read once + 12 B/row of pid
// traffic + the (partitions x blocks) histogram.
#include "common.cuh"
#include "primitives.cuh"
#include "multisplit.cuh"
#include "rtc.cuh"
#include "comm.cuh"
#include <memory>

namespace sb {

constexpr int MAX_KEYS = 8;
struct KeyCols {
  int n;
  int type[MAX_KEYS];
  const void *data[MAX_KEYS];
  const uint8_t *valid[MAX_KEYS];
  const int32_t *offs[MAX_KEYS];
};

// Murmur3Hash over the key columns of row i; NULL leaves the running hash unchanged (hash.scala:714),
// the running hash seeds the next column (hash.scala:400-409).
__device__ __forceinline__ uint32_t row_hash(const KeyCols &k, int64_t i, uint32_t seed) {
  uint32_t h = seed;
#pragma unroll 1
  for (int c = 0; c < k.n; c++) {
    if (!bit_valid(k.valid[c], i)) continue;
    switch (k.type[c]) {
      case SB_BOOL: h = mm3_int(((const uint8_t *)k.data[c])[i] ? 1u : 0u, h); break;
      case SB_INT8: h = mm3_int((uint32_t)(int32_t)((const int8_t *)k.data[c])[i], h); break;
      case SB_INT16: h = mm3_int((uint32_t)(int32_t)((const int16_t *)k.data[c])[i], h); break;
      case SB_INT32: case SB_DATE32: h = mm3_int(((const uint32_t *)k.data[c])[i], h); break;
      case SB_INT64: case SB_TIMESTAMP: case SB_DECIMAL64: h = mm3_long(((const uint64_t *)k.data[c])[i], h); break;
      case SB_FLOAT32: {
        float f = ((const float *)k.data[c])[i];
        h = mm3_int(f == 0.0f ? 0u : (uint32_t)float_bits_canonical(f), h);   // -0.0f -> 0 (hash.scala:718)
        break;
      }
      case SB_FLOAT64: {
        double d = ((const double *)k.data[c])[i];
        h = mm3_long(d == 0.0 ? 0ull : (uint64_t)double_bits_canonical(d), h);  // -0.0 -> 0 (hash.scala:720)
        break;
      }
      case SB_STRING: {
        int32_t o = k.offs[c][i], len = k.offs[c][i + 1] - o;
        h = mm3_bytes((const uint8_t *)k.data[c] + o, len, h);
        break;
      }
    }
  }
  return h;
}

// pmod (sql/api/.../catalyst/util/MathUtils.scala:96-99)
__device__ __forceinline__ int32_t pmod(int32_t a, int32_t n) {
  int32_t r = a % n;
  return r < 0 ? (r + n) % n : r;
}

constexpr int PART_THREADS = 256;
constexpr int PART_WARPS = PART_THREADS / 32;

// K1: pid + block histogram.  hist layout [partition][block].  key_mode: 0 = murmur3 hash of keys,
// 1 = round robin (pid = (start + 1 + i) mod n).
__global__ void __launch_bounds__(PART_THREADS) pid_hist_kernel(KeyCols keys, int64_t n, int32_t nparts, int64_t chunk,
                                                                int32_t *__restrict__ pid_out, uint32_t *__restrict__ hist,
                                                                int key_mode, int32_t rr_start) {
  extern __shared__ uint32_t sh_hist[];
  if (hist) {
    for (int p = threadIdx.x; p < nparts; p += PART_THREADS) sh_hist[p] = 0;
    __syncthreads();
  }
  int64_t begin = (int64_t)blockIdx.x * chunk;
  int64_t end = begin + chunk < n ? begin + chunk : n;
  for (int64_t i = begin + threadIdx.x; i < end; i += PART_THREADS) {
    int32_t p;
    if (key_mode == 0) p = pmod((int32_t)row_hash(keys, i, 42u), nparts);
    else p = (int32_t)(((int64_t)rr_start + 1 + i) % nparts);
    pid_out[i] = p;
    if (hist) atomicAdd(&sh_hist[p], 1u);
  }
  if (!hist) return;
  __syncthreads();
  for (int p = threadIdx.x; p < nparts; p += PART_THREADS) hist[(int64_t)p * gridDim.x + blockIdx.x] = sh_hist[p];
}

constexpr int SCATTER_MAX_COLS = 16;
constexpr int REMOTE_MAX_BUCKETS = 16;   // destinations of the fused exchange scatter (ranks on one NVSwitch domain)

// K2: stable multisplit of a group of columns with shared-memory regrouping (the scatter of an LSD radix sort pass,
// generalised to any set of fixed-width columns).  At most RG_MAX_NB buckets per pass; larger fan-outs run two passes
// (low digit, then high digit -- "LSB radix partition").
//
// This first kernel is the load/store version: it is what runs when a source column is not 16-byte aligned (the copy engine
// needs that) or with sb_config_set("regroup_ldst", 1); the default is regroup_tma_kernel further down, which shares phases A-D.
// A block owns a chunk of rows (one histogram column) and walks it in tiles of RGL_TILE rows.  Per tile:
//   A  every warp owns a contiguous 1/16 of the tile and walks it 32 rows at a time: same-bucket rows are ranked with
//      __match_any_sync + popcount on top of a per-warp shared-memory counter  -> (bucket, rank inside the warp's segment);
//   B  per bucket: exclusive prefix of the per-warp counts (order of the warps = order of the rows) and the tile total;
//   C  exclusive scan of the tile totals -> first sorted position of every bucket inside the tile;
//   D  every row now knows its position in the bucket-sorted tile; sorted position j knows its output row
//      gdest[j] = cursor[bucket] + (j - first[bucket]);
//   E  per column: coalesced global loads -> shared memory at the sorted position -> __syncthreads -> consecutive threads
//      read consecutive sorted positions and store them: rows of one bucket are adjacent, so the stores form RUNS
//      (tile/buckets rows long) instead of one LSU transaction and one partial-sector DRAM write per element
//      (a profile of the direct scatter showed several times the DRAM traffic of the data moved);
//   F  cursor[bucket] += tile total.
// Stability: positions are assigned in (bucket, row) order at every level, so arrival order is preserved per bucket.
constexpr int RGL_THREADS = 512;
constexpr int RGL_WARPS = RGL_THREADS / 32;
constexpr int RGL_ITEMS = 8;
constexpr int RGL_TILE = RGL_THREADS * RGL_ITEMS;   // 4096 rows
constexpr int RGL_SEG = RGL_TILE / RGL_WARPS;       // 256 rows per warp
constexpr int RG_MAX_NB = 256;
// The copy-engine kernel below comes in two tile sizes (the tile is also the granularity of the histograms): 512 threads x 4096
// rows, two blocks per SM -- best when the ranking phases dominate (sort passes, narrow rows, the 64 x 32 two-level split) -- and
// 1024 threads x 8192 rows, one block per SM -- runs twice as long and half as many sectors shared between tiles, best for wide
// rows into 100+ buckets (the big tiles slow a sort pass down).
constexpr int RG_ITEMS = 8;
constexpr int RG_TILE_SMALL = 512 * RG_ITEMS;
constexpr int RG_TILE_BIG = 1024 * RG_ITEMS;
constexpr int RG_SEG = 256;                      // rows per warp

struct RegroupCols {
  int ncols;
  int width[SCATTER_MAX_COLS];
  const void *src[SCATTER_MAX_COLS];
  void *dst[SCATTER_MAX_COLS];
  const uint8_t *src_valid[SCATTER_MAX_COLS];
  uint32_t *dst_valid[SCATTER_MAX_COLS];   // pre-set to all ones; NULL rows clear their bit
};

// one column of one tile: coalesced loads -> staging at the sorted position -> barrier -> run-forming stores.
// FULLT (tile completely populated) drops every predicate; addresses are base pointers + compile-time offsets.
template <typename T, bool FULLT>
__device__ __forceinline__ void regroup_move_column(const void *__restrict__ src, void *__restrict__ dst, int64_t first_row, int tid,
                                                    const uint32_t (&sp)[RGL_ITEMS], const uint32_t (&gdest)[RGL_ITEMS], uint32_t amask,
                                                    uint32_t gmask, uint64_t *staging) {
  const T *srcp = (const T *)src + first_row;       // row of item 0 for this lane; item `it` is 32 rows further
  T *stg = (T *)staging;
  const T *stg_read = (const T *)staging + tid;
  T v[RGL_ITEMS];
#pragma unroll
  for (int it = 0; it < RGL_ITEMS; it++)
    if (FULLT || ((amask >> it) & 1)) v[it] = __ldcs(srcp + it * 32);
#pragma unroll
  for (int it = 0; it < RGL_ITEMS; it++)
    if (FULLT || ((amask >> it) & 1)) stg[sp[it]] = v[it];
  __syncthreads();
#pragma unroll
  for (int it = 0; it < RGL_ITEMS; it++)
    if (FULLT || ((gmask >> it) & 1)) ((T *)dst)[gdest[it]] = stg_read[it * RGL_THREADS];
  __syncthreads();
}

__global__ void __launch_bounds__(RGL_THREADS, 2) regroup_kernel(const __grid_constant__ RegroupCols cols, const int32_t *__restrict__ bucket,
                                                                const uint32_t *__restrict__ base, int64_t n, int32_t nb, int64_t chunk,
                                                                int64_t *__restrict__ perm_out) {
  __shared__ __align__(16) uint64_t staging[RGL_TILE];      // 32 KB
  __shared__ uint8_t sbucket[RGL_TILE];                     // bucket of every sorted position (nb <= 256)
  __shared__ uint16_t wcnt[RGL_WARPS][RG_MAX_NB];
  __shared__ uint16_t first[RG_MAX_NB], tcnt[RG_MAX_NB];
  __shared__ uint32_t cursor[RG_MAX_NB];
  __shared__ uint32_t warp_sums[RGL_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t begin = (int64_t)blockIdx.x * chunk;
  const int64_t end = begin + chunk < n ? begin + chunk : n;
  for (int p = tid; p < nb; p += RGL_THREADS) cursor[p] = base[(int64_t)p * gridDim.x + blockIdx.x];
  for (int64_t tbase = begin; tbase < end; tbase += RGL_TILE) {
    const int tile_n = (int)(end - tbase < RGL_TILE ? end - tbase : RGL_TILE);
    const int64_t sbase = tbase + warp * RGL_SEG;     // first row of this warp's segment
    for (int p = lane; p < nb; p += 32) wcnt[warp][p] = 0;
    __syncwarp();
    // ---- A: rank inside the warp's segment --------------------------------------------------------------------------------
    uint32_t bl[RGL_ITEMS];   // low 16 bits: bucket (0xFFFF = no row); high 16 bits: rank in the warp segment, later sorted position
#pragma unroll
    for (int it = 0; it < RGL_ITEMS; it++) {
      const bool active = warp * RGL_SEG + it * 32 + lane < tile_n;
      const int32_t b = active ? __ldcs(bucket + sbase + it * 32 + lane) : -1 - lane;
      const uint32_t grp = __match_any_sync(0xffffffffu, b);
      const uint32_t rank = __popc(grp & lanemask_lt());
      uint32_t c = 0;
      if (active) {
        c = wcnt[warp][b];
        __syncwarp(grp);
        if (rank == 0) wcnt[warp][b] = (uint16_t)(c + __popc(grp));
      }
      __syncwarp();
      bl[it] = (active ? (uint32_t)b : 0xFFFFu) | ((c + rank) << 16);
    }
    __syncthreads();
    // ---- B: per bucket, exclusive prefix over the warps; tile total -------------------------------------------------------
    for (int p = tid; p < nb; p += RGL_THREADS) {
      uint32_t run = 0;
#pragma unroll
      for (int w = 0; w < RGL_WARPS; w++) {
        uint32_t c = wcnt[w][p];
        wcnt[w][p] = (uint16_t)run;
        run += c;
      }
      tcnt[p] = (uint16_t)run;
    }
    __syncthreads();
    // ---- C: exclusive scan of the tile totals -> first[] (nb <= 256: one bucket per thread of the first 8 warps) ------------
    {
      uint32_t v = tid < nb ? tcnt[tid] : 0, x = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
      }
      if (lane == 31) warp_sums[warp] = x;
      __syncthreads();
      uint32_t woff = 0;
      for (int w = 0; w < warp; w++) woff += warp_sums[w];
      if (tid < nb) first[tid] = (uint16_t)(woff + x - v);
    }
    __syncthreads();
    // ---- D: sorted position of every row; bucket of every sorted position --------------------------------------------------
#pragma unroll
    for (int it = 0; it < RGL_ITEMS; it++) {
      const uint32_t b = bl[it] & 0xFFFFu;
      if (b != 0xFFFFu) {
        const uint32_t sp = first[b] + wcnt[warp][b] + (bl[it] >> 16);
        sbucket[sp] = (uint8_t)b;
        bl[it] = b | (sp << 16);
      }
    }
    __syncthreads();
    uint32_t gdest[RGL_ITEMS];    // output row of sorted position j = it * RGL_THREADS + tid
    uint32_t sp[RGL_ITEMS];       // sorted position of this thread's rows
    uint32_t amask = 0, gmask = 0;
#pragma unroll
    for (int it = 0; it < RGL_ITEMS; it++) {
      const int j = it * RGL_THREADS + tid;
      if (j < tile_n) {
        const int b = sbucket[j];
        gdest[it] = cursor[b] + (uint32_t)(j - first[b]);
        gmask |= 1u << it;
      } else gdest[it] = 0;
      sp[it] = bl[it] >> 16;
      if ((bl[it] & 0xFFFFu) != 0xFFFFu) amask |= 1u << it;
    }
    const bool fullt = tile_n == RGL_TILE;
    const int64_t first_row = sbase + lane;
    // ---- E: move the columns -----------------------------------------------------------------------------------------------
    if (perm_out) {   // row ids travel like a column (used to gather variable-width columns afterwards)
#pragma unroll
      for (int it = 0; it < RGL_ITEMS; it++)
        if ((amask >> it) & 1) staging[sp[it]] = (uint64_t)(first_row + it * 32);
      __syncthreads();
#pragma unroll
      for (int it = 0; it < RGL_ITEMS; it++)
        if ((gmask >> it) & 1) perm_out[gdest[it]] = (int64_t)staging[it * RGL_THREADS + tid];
      __syncthreads();
    }
#pragma unroll 1
    for (int c = 0; c < cols.ncols; c++) {
      const int w = cols.width[c];
      const void *src = cols.src[c];
      void *dst = cols.dst[c];
      {   // pull the NEXT column's rows of this tile (or the next tile's bucket ids) towards L2 while this column moves
        const bool last = c + 1 == cols.ncols;
        const char *nsrc = last ? (const char *)(bucket + RGL_TILE) : (const char *)cols.src[c + 1];
        const int nw = last ? 4 : cols.width[c + 1];
        if (!last || tbase + RGL_TILE + RGL_TILE <= end) {
#pragma unroll
          for (int it = 0; it < RGL_ITEMS; it++)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(nsrc + (first_row + it * 32) * nw));
        }
      }
#define SB_REGROUP(T)                                                                                              \
  if (fullt) regroup_move_column<T, true>(src, dst, first_row, tid, sp, gdest, amask, gmask, staging);              \
  else regroup_move_column<T, false>(src, dst, first_row, tid, sp, gdest, amask, gmask, staging);
      switch (w) {
        case 1: SB_REGROUP(uint8_t) break;
        case 2: SB_REGROUP(uint16_t) break;
        case 4: SB_REGROUP(uint32_t) break;
        default: SB_REGROUP(uint64_t) break;
      }
#undef SB_REGROUP
      if (cols.dst_valid[c]) {   // NULLs: clear the destination bit (rare, scattered)
        const uint8_t *sv = cols.src_valid[c];
#pragma unroll
        for (int it = 0; it < RGL_ITEMS; it++) {
          if (!((amask >> it) & 1)) continue;
          if (!bit_valid(sv, first_row + it * 32)) {
            const uint32_t b = sbucket[sp[it]];
            const uint32_t d = cursor[b] + (sp[it] - first[b]);
            atomicAnd(&cols.dst_valid[c][d >> 5], ~(1u << (d & 31)));
          }
        }
      }
    }
    __syncthreads();
    // ---- F: advance the block's cursors ----------------------------------------------------------------------------------------
    for (int p = tid; p < nb; p += RGL_THREADS) cursor[p] += tcnt[p];
    __syncthreads();
  }
}

// ---- K2, copy-engine version -------------------------------------------------------------------------------------------------
// Same tile algebra as regroup_kernel (phases A-D, F), but phase E no longer loads anything itself: one elected thread keeps
// RGT_STAGES bulk copies (cp.async.bulk -> mbarrier) in flight per block, walking the sequence
//   tile 0: [bucket ids, column 0, column 1, ...], tile 1: [...], ...
// so the next column tiles stream into shared memory in ROW order while the warps drain the current one.  Draining is
// output-driven: the thread that owns sorted position j knows which row of the tile lands there (src = inverse of the
// tile's bucket-sort permutation, kept in registers) and where it goes (gdest), so a column costs one shared-memory gather
// and one global store per row and a single __syncthreads() (to hand the stage back), instead of
// "global load -> shared scatter -> barrier -> shared load -> global store -> barrier" with the load latency exposed.
constexpr int RGT_STAGES = 3;

template <typename T, bool FULLT>
__device__ __forceinline__ void regroup_drain_column(const uint8_t *__restrict__ stage, void *__restrict__ dst,
                                                     const uint32_t (&src2)[RG_ITEMS / 2], const uint32_t (&gdest)[RG_ITEMS],
                                                     uint32_t gmask) {
  const T *s = (const T *)stage;
  T v[RG_ITEMS];
#pragma unroll
  for (int it = 0; it < RG_ITEMS; it++) v[it] = s[(src2[it >> 1] >> ((it & 1) * 16)) & 0xFFFFu];
#pragma unroll
  for (int it = 0; it < RG_ITEMS; it++)
    if (FULLT || ((gmask >> it) & 1)) ((T *)dst)[gdest[it]] = v[it];
}

// REMOTE drain: the run of bucket b goes to bucket b's OWN base address (a peer GPU's receive window mapped over NVLink, or
// this GPU's own window): ptrs[b] is pre-biased so that the element for global sorted position g lands at ptrs[b] + g * sizeof(T).
template <typename T, bool FULLT>
__device__ __forceinline__ void regroup_drain_column_remote(const uint8_t *__restrict__ stage, const uint64_t *__restrict__ ptrs,
                                                            const uint32_t (&src2)[RG_ITEMS / 2], const uint32_t (&gdest)[RG_ITEMS],
                                                            const uint32_t (&bk2)[RG_ITEMS / 4], uint32_t gmask) {
  const T *s = (const T *)stage;
  T v[RG_ITEMS];
#pragma unroll
  for (int it = 0; it < RG_ITEMS; it++) v[it] = s[(src2[it >> 1] >> ((it & 1) * 16)) & 0xFFFFu];
#pragma unroll
  for (int it = 0; it < RG_ITEMS; it++)
    if (FULLT || ((gmask >> it) & 1)) {
      T *dst = (T *)(uintptr_t)ptrs[(bk2[it >> 2] >> ((it & 3) * 8)) & 0xFFu];
      dst[gdest[it]] = v[it];
    }
}

// REMOTE = the fused exchange scatter (sb_shuffle_exchange): buckets are destination ranks and every bucket's rows are stored
// straight into that rank's receive window (`bptr`: [ncols][nb] pre-biased byte addresses) -- the multisplit IS the transport.
template <int RG_THREADS, bool REMOTE = false>
__global__ void __launch_bounds__(RG_THREADS, 1024 / RG_THREADS) regroup_tma_kernel(const __grid_constant__ RegroupCols cols, const int32_t *__restrict__ bucket,
                                                                                 const uint32_t *__restrict__ base, int64_t n, int32_t nb, int64_t ntiles,
                                                                                 int64_t *__restrict__ perm_out, int l2_stream,
                                                                                 const uint64_t *__restrict__ bptr = nullptr) {
  constexpr int RG_WARPS = RG_THREADS / 32, RG_TILE = RG_THREADS * RG_ITEMS;
  constexpr int RGT_STAGE_BYTES = RG_TILE * 8;   // one 8-byte column tile
  static_assert(RG_TILE / RG_WARPS == RG_SEG, "a warp ranks 256 rows");
  extern __shared__ __align__(128) uint8_t ring[];          // RGT_STAGES x RGT_STAGE_BYTES
  __shared__ __align__(8) uint64_t bars[RGT_STAGES];
  __shared__ uint32_t readers_done[RGT_STAGES];
  // wcnt (phases A-D) and ssrc (D-E) share storage; nothing but the copy engine ever writes a full stage, so handing a stage back
  // needs no proxy fence (a fence.proxy.async is a MEMBAR.ALL.CTA: it would wait for the column's global stores to drain)
  __shared__ __align__(16) uint16_t wcnt_ssrc[RG_TILE];
  __shared__ uint8_t sbucket[RG_TILE];
  __shared__ uint16_t first[RG_MAX_NB], tcnt[RG_MAX_NB];
  uint16_t (*wcnt)[RG_MAX_NB] = reinterpret_cast<uint16_t (*)[RG_MAX_NB]>(wcnt_ssrc);
  uint16_t *ssrc = wcnt_ssrc;
  static_assert(RG_WARPS * RG_MAX_NB <= RG_TILE, "wcnt must fit in the ssrc storage");
  __shared__ uint32_t cursor[RG_MAX_NB];
  __shared__ uint32_t warp_sums[RG_WARPS];
  __shared__ uint64_t s_bptr[REMOTE ? SCATTER_MAX_COLS * REMOTE_MAX_BUCKETS : 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (REMOTE)
    for (int i = tid; i < cols.ncols * nb; i += RG_THREADS) s_bptr[i] = bptr[i];
  // Tiles are dealt round-robin (block b: tiles b, b + grid, ...), so at any moment the grid works on ~grid CONSECUTIVE tiles:
  // their runs are adjacent inside every bucket, which lets L2 complete the sectors two tiles share before eviction and keeps
  // the DRAM write stream to (buckets x columns) compact regions instead of (blocks x buckets x columns) scattered ones.
  if ((int64_t)blockIdx.x >= ntiles) return;
  const int64_t tstride = (int64_t)gridDim.x * RG_TILE;
  const int64_t begin = (int64_t)blockIdx.x * RG_TILE;
  const int64_t end = n;
  const int per_tile = cols.ncols + 1;
  // Item i of the block's sequence (tile-major, [bucket ids, columns...] inside a tile) lives in stage i % RGT_STAGES.  A stage is
  // refilled by whichever WARP finishes reading it last (shared counter), so the column loop has no block-wide barrier: warps
  // drift up to RGT_STAGES - 1 items apart and a fast warp never waits for a slow one, only for data.
  auto issue = [&](int64_t tb, int q, int stg_i) {
    while (q >= per_tile) {
      q -= per_tile;
      tb += tstride;
    }
    if (tb >= end) return;
    const int64_t rows = end - tb < RG_TILE ? end - tb : RG_TILE;
    const char *src;
    int w;
    if (q == 0) {
      src = (const char *)(bucket + tb);
      w = 4;
    } else {
      w = cols.width[q - 1];
      src = (const char *)cols.src[q - 1] + tb * w;
    }
    const uint32_t bytes = (uint32_t)(rows * w) & ~15u;     // a ragged tail (< 16 B) is fetched by the consumers
    if (bytes) {
      mbar_arrive_expect_tx(&bars[stg_i], bytes);
      if (l2_stream) tma_load_1d_stream(ring + stg_i * RGT_STAGE_BYTES, src, bytes, &bars[stg_i]);
      else tma_load_1d(ring + stg_i * RGT_STAGE_BYTES, src, bytes, &bars[stg_i]);
    } else {
      mbar_arrive(&bars[stg_i]);
    }
  };
  if (tid == 0) {
    for (int i = 0; i < RGT_STAGES; i++) {
      mbar_init(&bars[i], 1);
      readers_done[i] = 0;
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async_smem();
  }
  __syncthreads();
  if (tid == 0)
    for (int i = 0; i < RGT_STAGES; i++) issue(begin, i, i);
  int stage = 0;
  uint32_t phase = 0;
  // waits for the current stage; fetches the ragged tail of a partial tile; returns the stage's base
  auto acquire = [&](const void *col_base, int w, int64_t tbase, int tile_n) -> uint8_t * {
    mbar_wait(&bars[stage], phase);
    uint8_t *stg = ring + stage * RGT_STAGE_BYTES;
    if (tile_n < RG_TILE) {
      const uint32_t total = (uint32_t)tile_n * w, done = total & ~15u;
      if (tid < (int)(total - done)) stg[done + tid] = ((const uint8_t *)col_base + tbase * w)[done + tid];
      fence_proxy_async_smem();   // generic-proxy bytes in a stage the copy engine will overwrite later
      __syncthreads();
    }
    return stg;
  };
  // this warp is done with item (tbase, q) in the current stage; the last warp to say so refills the stage with item + RGT_STAGES
  auto release = [&](int64_t tbase, int q) {
    __syncwarp();
    if (lane == 0 && (smem_add_acq_rel(&readers_done[stage], 1) + 1) % RG_WARPS == 0)   // never reset: RG_WARPS arrivals per use
      issue(tbase, q + RGT_STAGES, stage);
    if (++stage == RGT_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  };
  int64_t tile = blockIdx.x;
  for (int64_t tbase = begin; tbase < end; tbase += tstride, tile += gridDim.x) {
    const int tile_n = (int)(end - tbase < RG_TILE ? end - tbase : RG_TILE);
    const bool fullt = tile_n == RG_TILE;
    // first output row of every bucket for THIS tile (read by phase D, several barriers from here; the previous tile's readers
    // are behind the barrier that ended its register load)
    for (int p = tid; p < nb; p += RG_THREADS) cursor[p] = base[(int64_t)p * ntiles + tile];
    for (int p = lane; p < nb; p += 32) wcnt[warp][p] = 0;
    __syncwarp();
    const uint8_t *stg = acquire(bucket, 4, tbase, tile_n);
    // ---- A: rank inside the warp's segment (bucket ids come from the stage) ------------------------------------------------
    uint32_t bl[RG_ITEMS];
    {
      const int32_t *sb = (const int32_t *)stg + warp * RG_SEG + lane;
#pragma unroll
      for (int it = 0; it < RG_ITEMS; it++) {
        const bool active = warp * RG_SEG + it * 32 + lane < tile_n;
        const int32_t b = active ? sb[it * 32] : -1 - lane;
        const uint32_t grp = __match_any_sync(0xffffffffu, b);
        const uint32_t rank = __popc(grp & lanemask_lt());
        uint32_t c = 0;
        if (active) {
          c = wcnt[warp][b];
          __syncwarp(grp);
          if (rank == 0) wcnt[warp][b] = (uint16_t)(c + __popc(grp));
        }
        __syncwarp();
        bl[it] = (active ? (uint32_t)b : 0xFFFFu) | ((c + rank) << 16);
      }
    }
    release(tbase, 0);   // this warp has consumed its bucket ids
    __syncthreads();
    // ---- B: per bucket, exclusive prefix over the warps; tile total -------------------------------------------------------
    for (int p = tid; p < nb; p += RG_THREADS) {
      uint32_t run = 0;
#pragma unroll
      for (int w = 0; w < RG_WARPS; w++) {
        uint32_t c = wcnt[w][p];
        wcnt[w][p] = (uint16_t)run;
        run += c;
      }
      tcnt[p] = (uint16_t)run;
    }
    __syncthreads();
    // ---- C: exclusive scan of the tile totals -> first[] -------------------------------------------------------------------
    {
      uint32_t v = tid < nb ? tcnt[tid] : 0, x = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
      }
      if (lane == 31) warp_sums[warp] = x;
      __syncthreads();
      uint32_t woff = 0;
      for (int w = 0; w < warp; w++) woff += warp_sums[w];
      if (tid < nb) first[tid] = (uint16_t)(woff + x - v);
    }
    __syncthreads();
    // ---- D: sorted position of every row -> (bucket, source row) of every sorted position ---------------------------------------
#pragma unroll
    for (int it = 0; it < RG_ITEMS; it++) {
      const uint32_t b = bl[it] & 0xFFFFu;
      if (b != 0xFFFFu) bl[it] = b | ((first[b] + wcnt[warp][b] + (bl[it] >> 16)) << 16);
    }
    __syncthreads();    // wcnt is dead: ssrc may overwrite it
#pragma unroll
    for (int it = 0; it < RG_ITEMS; it++) {
      const uint32_t b = bl[it] & 0xFFFFu;
      if (b != 0xFFFFu) {
        sbucket[bl[it] >> 16] = (uint8_t)b;
        ssrc[bl[it] >> 16] = (uint16_t)(warp * RG_SEG + it * 32 + lane);
      }
    }
    __syncthreads();
    uint32_t gdest[RG_ITEMS];        // output row of sorted position j = it * RG_THREADS + tid
    uint32_t src2[RG_ITEMS / 2];     // tile row that lands at sorted position j, two per register
    uint32_t bk2[RG_ITEMS / 4] = {0};   // REMOTE: bucket of sorted position j, four per register
    uint32_t gmask = 0;
#pragma unroll
    for (int it = 0; it < RG_ITEMS; it++) {
      const int j = it * RG_THREADS + tid;
      uint32_t srow = 0;
      if (j < tile_n) {
        const int b = sbucket[j];
        gdest[it] = cursor[b] + (uint32_t)(j - first[b]);
        srow = ssrc[j];
        gmask |= 1u << it;
        if (REMOTE) bk2[it >> 2] |= (uint32_t)b << ((it & 3) * 8);
      } else gdest[it] = 0;
      if (it & 1) src2[it >> 1] |= srow << 16;
      else src2[it >> 1] = srow;
    }
    __syncthreads();    // ssrc is in registers: the next tile may zero wcnt
    // ---- E: drain the columns ------------------------------------------------------------------------------------------------
    if (perm_out) {   // row ids of the rows in output order (used to gather variable-width columns afterwards)
#pragma unroll
      for (int it = 0; it < RG_ITEMS; it++)
        if ((gmask >> it) & 1) perm_out[gdest[it]] = tbase + (int64_t)((src2[it >> 1] >> ((it & 1) * 16)) & 0xFFFFu);
    }
#pragma unroll 1
    for (int c = 0; c < cols.ncols; c++) {
      const int w = cols.width[c];
      void *dst = cols.dst[c];
      const uint8_t *cs = acquire(cols.src[c], w, tbase, tile_n);
#define SB_DRAIN(T)                                                                                            \
  if (REMOTE) {                                                                                                \
    if (fullt) regroup_drain_column_remote<T, true>(cs, s_bptr + c * nb, src2, gdest, bk2, gmask);           \
    else regroup_drain_column_remote<T, false>(cs, s_bptr + c * nb, src2, gdest, bk2, gmask);                \
  } else if (fullt) regroup_drain_column<T, true>(cs, dst, src2, gdest, gmask);                              \
  else regroup_drain_column<T, false>(cs, dst, src2, gdest, gmask);
      switch (w) {
        case 1: SB_DRAIN(uint8_t) break;
        case 2: SB_DRAIN(uint16_t) break;
        case 4: SB_DRAIN(uint32_t) break;
        default: SB_DRAIN(uint64_t) break;
      }
#undef SB_DRAIN
      if (!REMOTE && cols.dst_valid[c]) {   // NULLs: clear the destination bit (rare, scattered)
        const uint8_t *sv = cols.src_valid[c];
#pragma unroll
        for (int it = 0; it < RG_ITEMS; it++) {
          if (!((gmask >> it) & 1)) continue;
          const int64_t row = tbase + (int64_t)((src2[it >> 1] >> ((it & 1) * 16)) & 0xFFFFu);
          if (!bit_valid(sv, row)) atomicAnd(&cols.dst_valid[c][gdest[it] >> 5], ~(1u << (gdest[it] & 31)));
        }
      }
      release(tbase, c + 1);
    }
  }
}

// bucket = digit of a partition id for the two-level split; also the per-block histogram in multisplit layout
constexpr int PDH_THREADS = 512;
__global__ void __launch_bounds__(PDH_THREADS) pid_digit_hist_kernel(const int32_t *__restrict__ pid, int64_t n, int32_t div, int32_t mod,
                                                                    int32_t nb, int64_t chunk, int32_t *__restrict__ bucket,
                                                                    uint32_t *__restrict__ hist) {
  __shared__ uint32_t sh[RG_MAX_NB];
  for (int p = threadIdx.x; p < nb; p += PDH_THREADS) sh[p] = 0;
  __syncthreads();
  int64_t begin = (int64_t)blockIdx.x * chunk;
  int64_t end = begin + chunk < n ? begin + chunk : n;
  for (int64_t i = begin + threadIdx.x; i < end; i += PDH_THREADS) {
    int b = (pid[i] / div) % mod;
    bucket[i] = b;
    atomicAdd(&sh[b], 1u);
  }
  __syncthreads();
  for (int p = threadIdx.x; p < nb; p += PDH_THREADS) hist[(int64_t)p * gridDim.x + blockIdx.x] = sh[p];
}

__global__ void part_offsets_kernel(const uint32_t *__restrict__ base, int32_t nparts, int nblocks, int64_t n,
                                    int64_t *__restrict__ out_offsets) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < nparts) out_offsets[p] = base[(int64_t)p * nblocks];
  if (p == nparts) out_offsets[p] = n;
}

static KeyCols make_keys(const sb_table *in, const int32_t *key_cols, int32_t nkeys) {
  SB_REQUIRE(nkeys >= 0 && nkeys <= MAX_KEYS, "at most %d partitioning keys are supported (got %d)", MAX_KEYS, nkeys);
  KeyCols k;
  k.n = nkeys;
  for (int i = 0; i < nkeys; i++) {
    SB_REQUIRE(key_cols[i] >= 0 && key_cols[i] < (int)in->cols.size(), "key column %d out of range", key_cols[i]);
    const Column &c = in->cols[key_cols[i]];
    k.type[i] = c.type;
    k.data[i] = c.d();
    k.valid[i] = c.v();
    k.offs[i] = c.o();
  }
  return k;
}

PartGeometry part_geometry(int64_t n, int32_t nbuckets, bool big_tiles) {
  PartGeometry g;
  if (nbuckets <= RG_MAX_NB) {
    // one histogram column per TILE: the scatter deals tiles round-robin to a persistent grid (see regroup_tma_kernel)
    g.chunk = big_tiles ? RG_TILE_BIG : RG_TILE_SMALL;
    int64_t nt = (n + g.chunk - 1) / g.chunk;
    g.nblocks = (int)(nt < 1 ? 1 : nt);
    return g;
  }
  // above the single-pass fan-out the caller's histogram only provides the bucket boundaries: keep it coarse
  const int64_t T = RG_TILE_SMALL;
  int64_t want = (n + T * 2 - 1) / (T * 2);
  int maxb = rt().num_sms * 2;
  g.nblocks = (int)(want < 1 ? 1 : (want > maxb ? maxb : want));
  g.chunk = ((n + g.nblocks - 1) / g.nblocks + T - 1) / T * T;
  if (g.chunk < T) g.chunk = T;
  g.nblocks = (int)((n + g.chunk - 1) / g.chunk);
  if (g.nblocks < 1) g.nblocks = 1;
  return g;
}

static void regroup_pass(const int32_t *bucket_dev, uint32_t *hist_dev, int32_t nb, const PartGeometry &g, const SplitCol *cols,
                         int ncols, int64_t n, int64_t *perm_out, int64_t *offsets_dev, cudaStream_t st) {
  exclusive_scan_i32((const int32_t *)hist_dev, (int32_t *)hist_dev, (int64_t)nb * g.nblocks, nullptr, st);
  if (offsets_dev) {
    part_offsets_kernel<<<(nb + 1 + 255) / 256, 256, 0, st>>>(hist_dev, nb, g.nblocks, n, offsets_dev);
    SB_LAUNCH_CHECK();
  }
  if (n == 0) return;
  SB_REQUIRE(g.chunk == RG_TILE_SMALL || g.chunk == RG_TILE_BIG, "internal: regroup needs a per-tile histogram");
  const bool big = g.chunk == RG_TILE_BIG;
  int done = 0;
  bool first = true;
  while (first || done < ncols) {
    RegroupCols rc;
    rc.ncols = 0;
    const int max_cols = SCATTER_MAX_COLS;
    const int l2_stream = 0;
    while (done < ncols && rc.ncols < max_cols) {
      const SplitCol &c = cols[done++];
      int k = rc.ncols++;
      rc.width[k] = c.width;
      rc.src[k] = c.src;
      rc.dst[k] = c.dst;
      rc.src_valid[k] = c.src_valid;
      rc.dst_valid[k] = c.dst_valid;
    }
    if (rc.ncols > 0 || (first && perm_out)) {
      // the copy engine wants 16-byte aligned sources; anything else (a caller-provided, oddly offset device buffer) takes the
      // load/store kernel.  sb_config_set("regroup_ldst", 1) forces it; the shuffle tests of tests/test_gpu_row_movement.py run
      // with both settings, and a source borrowed one element past an aligned allocation takes it whatever the setting.
      const bool force_ldst = config().regroup_ldst != 0;
      bool aligned = ((uintptr_t)bucket_dev & 15) == 0;
      for (int k = 0; k < rc.ncols; k++) aligned = aligned && ((uintptr_t)rc.src[k] & 15) == 0;
      KernelTimer kt("partition_scatter", st);
      if (aligned && !force_ldst) {
        static std::once_flag once;
        std::call_once(once, [] {
          SB_CUDA(cudaFuncSetAttribute(regroup_tma_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, RGT_STAGES * RG_TILE_SMALL * 8));
          SB_CUDA(cudaFuncSetAttribute(regroup_tma_kernel<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, RGT_STAGES * RG_TILE_BIG * 8));
        });
        const int bps = big ? 1 : 2;
        const int grid = g.nblocks < rt().num_sms * bps ? g.nblocks : rt().num_sms * bps;
        if (big)
          regroup_tma_kernel<1024><<<grid, 1024, RGT_STAGES * RG_TILE_BIG * 8, st>>>(rc, bucket_dev, hist_dev, n, nb, (int64_t)g.nblocks,
                                                                                  first ? perm_out : nullptr, l2_stream);
        else
          regroup_tma_kernel<512><<<grid, 512, RGT_STAGES * RG_TILE_SMALL * 8, st>>>(rc, bucket_dev, hist_dev, n, nb, (int64_t)g.nblocks,
                                                                                  first ? perm_out : nullptr, l2_stream);
      } else {
        regroup_kernel<<<g.nblocks, RGL_THREADS, 0, st>>>(rc, bucket_dev, hist_dev, n, nb, g.chunk, first ? perm_out : nullptr);
      }
      SB_LAUNCH_CHECK();
    }
    first = false;
  }
}

void multisplit_scatter(const int32_t *bucket_dev, uint32_t *hist_dev, int32_t nbuckets, const PartGeometry &g,
                        const SplitCol *cols, int ncols, int64_t n, int64_t *perm_out, int64_t *offsets_dev,
                        cudaStream_t st) {
  SB_REQUIRE(nbuckets >= 1 && nbuckets <= MULTISPLIT_MAX_BUCKETS, "multisplit supports up to %d buckets (got %d)",
             MULTISPLIT_MAX_BUCKETS, nbuckets);
  SB_REQUIRE(n < 0xFFFFFFFFll, "tables of 2^32 rows or more must be split in chunks");
  if (nbuckets <= RG_MAX_NB) {
    regroup_pass(bucket_dev, hist_dev, nbuckets, g, cols, ncols, n, perm_out, offsets_dev, st);
    return;
  }
  // ---- two-level LSB split: pass 1 on the low digit (bucket % B1), pass 2 on the high digit (bucket / B1).  Both passes
  // are stable, so the result is ordered by (high, low) = bucket id with arrival order preserved inside a bucket.
  const int32_t B1 = 64, B2 = (nbuckets + B1 - 1) / B1;
  SB_REQUIRE(B2 <= RG_MAX_NB, "too many buckets");
  const PartGeometry g2 = part_geometry(n, RG_MAX_NB, false);   // per-tile histograms for the two digit passes
  Scratch digit(n * 4 + 16, st), hist2((int64_t)RG_MAX_NB * g2.nblocks * 4 + 16, st), pid_mid(n * 4 + 16, st), perm_mid(perm_out ? n * 8 + 16 : 0, st);
  // intermediate copies of every column (+ validity carried as-is through atomicAnd on a fresh bitmap)
  std::vector<SplitCol> c1(cols, cols + ncols), c2(cols, cols + ncols);
  std::vector<Scratch *> tmp;
  struct Guard {
    std::vector<Scratch *> &t;
    ~Guard() { for (auto *x : t) delete x; }
  } guard{tmp};
  for (int i = 0; i < ncols; i++) {
    Scratch *d = new Scratch((int64_t)n * cols[i].width + 16, st);
    tmp.push_back(d);
    c1[i].dst = d->ptr;
    c2[i].src = d->ptr;
    if (cols[i].dst_valid) {
      Scratch *v = new Scratch(bitmap_alloc_bytes(n), st);
      tmp.push_back(v);
      SB_CUDA(cudaMemsetAsync(v->ptr, 0xff, (size_t)bitmap_alloc_bytes(n), st));
      c1[i].dst_valid = (uint32_t *)v->ptr;
      c2[i].src_valid = (const uint8_t *)v->ptr;
    }
  }
  c1.push_back({4, bucket_dev, pid_mid.ptr, nullptr, nullptr});   // the bucket ids travel with the rows into pass 2
  if (n > 0) {
    pid_digit_hist_kernel<<<g2.nblocks, PDH_THREADS, 0, st>>>(bucket_dev, n, 1, B1, B1, g2.chunk, digit.as<int32_t>(), hist2.as<uint32_t>());
    SB_LAUNCH_CHECK();
  }
  regroup_pass(digit.as<int32_t>(), hist2.as<uint32_t>(), B1, g2, c1.data(), (int)c1.size(), n, perm_out ? perm_mid.as<int64_t>() : nullptr, nullptr, st);
  if (perm_out) c2.push_back({8, perm_mid.ptr, perm_out, nullptr, nullptr});
  if (n > 0) {
    pid_digit_hist_kernel<<<g2.nblocks, PDH_THREADS, 0, st>>>(pid_mid.as<int32_t>(), n, B1, B2, B2, g2.chunk, digit.as<int32_t>(), hist2.as<uint32_t>());
    SB_LAUNCH_CHECK();
  }
  regroup_pass(digit.as<int32_t>(), hist2.as<uint32_t>(), B2, g2, c2.data(), (int)c2.size(), n, nullptr, nullptr, st);
  // bucket boundaries come from the caller's full-resolution histogram
  exclusive_scan_i32((const int32_t *)hist_dev, (int32_t *)hist_dev, (int64_t)nbuckets * g.nblocks, nullptr, st);
  if (offsets_dev) {
    part_offsets_kernel<<<(nbuckets + 1 + 255) / 256, 256, 0, st>>>(hist_dev, nbuckets, g.nblocks, n, offsets_dev);
    SB_LAUNCH_CHECK();
  }
  SB_CUDA(cudaStreamSynchronize(st));   // temporaries are released by the guard
}

// mode 0 = hash, 1 = round robin
static void partition_impl(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t nparts, int mode,
                           int32_t rr_start, cudaStream_t st, sb_table **out, int64_t *out_offsets_host) {
  SB_REQUIRE(in && out && out_offsets_host, "null argument");
  SB_REQUIRE(nparts >= 1, "num_partitions must be >= 1");
  int64_t n = in->nrows;
  if (nparts > MULTISPLIT_MAX_BUCKETS)
    fail(SB_ERR_UNSUPPORTED, "num_partitions %d exceeds the single-pass multisplit limit (%d)", nparts, MULTISPLIT_MAX_BUCKETS);
  KeyCols keys;
  keys.n = 0;
  if (mode == 0) keys = make_keys(in, key_cols, nkeys);
  int64_t rowbytes = 0;
  auto by_row_id = [](const Column &c) { return c.type == SB_STRING || c.type == SB_DECIMAL128; };   // moved by one gather at the end
  for (auto &c : in->cols) rowbytes += by_row_id(c) ? 8 : type_width(c.type);
  const bool big_tiles = nparts >= 64 && rowbytes >= 32;
  PartGeometry g = part_geometry(n, nparts, big_tiles);
  Scratch pid(n * 4 + 16, st);
  Scratch hist((int64_t)nparts * g.nblocks * 4 + 16, st);
  Scratch offs_dev((nparts + 1) * 8, st);
  static bool attr_set = false;
  if (!attr_set) {
    SB_CUDA(cudaFuncSetAttribute(pid_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  pid_hist_kernel<<<g.nblocks, PART_THREADS, (size_t)nparts * 4, st>>>(keys, n, nparts, g.chunk, pid.as<int32_t>(),
                                                                        hist.as<uint32_t>(), mode, rr_start);
  SB_LAUNCH_CHECK();

  sb_table *t = table_new(n);
  try {
    bool need_perm = false;
    for (auto &c : in->cols) need_perm |= by_row_id(c);
    Scratch perm(need_perm ? n * 8 + 8 : 0, st);
    t->cols.resize(in->cols.size());
    std::vector<SplitCol> sc;
    for (size_t i = 0; i < in->cols.size(); i++) {
      const Column &c = in->cols[i];
      if (by_row_id(c)) continue;
      Column r = column_alloc(c.type, c.scale, n, c.validity != nullptr, st);
      if (r.validity) SB_CUDA(cudaMemsetAsync(r.validity->ptr, 0xff, (size_t)bitmap_alloc_bytes(n), st));
      r.null_count = c.null_count;
      t->cols[i] = r;
      sc.push_back({type_width(c.type), c.d(), r.data->ptr, c.v(), r.validity ? (uint32_t *)r.validity->ptr : nullptr});
    }
    multisplit_scatter(pid.as<int32_t>(), hist.as<uint32_t>(), nparts, g, sc.data(), (int)sc.size(), n,
                       need_perm ? perm.as<int64_t>() : nullptr, offs_dev.as<int64_t>(), st);
    if (need_perm) {
      for (size_t i = 0; i < in->cols.size(); i++)
        if (by_row_id(in->cols[i])) t->cols[i] = gather_column(in->cols[i], perm.as<int64_t>(), n, false, st);
    }
    SB_CUDA(cudaMemcpyAsync(out_offsets_host, offs_dev.ptr, (size_t)(nparts + 1) * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
}

// ---- fused exchange: the multisplit IS the transport ----------------------------------------------------------------------------
// destination rank of every row (owner of its partition id: contiguous ownership ranges) + the per-tile histogram over ranks
struct OwnerBounds { int32_t first[REMOTE_MAX_BUCKETS + 1]; };   // rank r owns partitions [first[r], first[r + 1])
__global__ void __launch_bounds__(PDH_THREADS) owner_hist_kernel(const int32_t *__restrict__ pid, int64_t n, OwnerBounds ob, int32_t nranks, int64_t chunk,
                                                                 int32_t *__restrict__ bucket, uint32_t *__restrict__ hist) {
  __shared__ uint32_t sh[REMOTE_MAX_BUCKETS];
  if (threadIdx.x < REMOTE_MAX_BUCKETS) sh[threadIdx.x] = 0;
  __syncthreads();
  const int64_t begin = (int64_t)blockIdx.x * chunk, end = begin + chunk < n ? begin + chunk : n;
  for (int64_t i = begin + threadIdx.x; i < end; i += PDH_THREADS) {
    const int32_t p = pid[i];
    int d = 0;
#pragma unroll 1
    for (int r = 1; r < nranks; r++) d += p >= ob.first[r];
    bucket[i] = d;
    atomicAdd(&sh[d], 1u);
  }
  __syncthreads();
  if (threadIdx.x < nranks) hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = sh[threadIdx.x];
}
// local partition index (pid - first owned partition) of every received row + per-tile histogram in multisplit layout
__global__ void __launch_bounds__(PDH_THREADS) local_pid_hist_kernel(const int32_t *__restrict__ pid, int64_t n, int32_t lo, int32_t nb, int64_t chunk,
                                                                     int32_t *__restrict__ bucket, uint32_t *__restrict__ hist) {
  extern __shared__ uint32_t lph_sh[];
  for (int p = threadIdx.x; p < nb; p += PDH_THREADS) lph_sh[p] = 0;
  __syncthreads();
  const int64_t begin = (int64_t)blockIdx.x * chunk, end = begin + chunk < n ? begin + chunk : n;
  for (int64_t i = begin + threadIdx.x; i < end; i += PDH_THREADS) {
    const int32_t b = pid[i] - lo;
    bucket[i] = b;
    atomicAdd(&lph_sh[b], 1u);
  }
  __syncthreads();
  for (int p = threadIdx.x; p < nb; p += PDH_THREADS) hist[(int64_t)p * gridDim.x + blockIdx.x] = lph_sh[p];
}

static inline int32_t owner_first(int32_t r, int32_t nparts, int32_t nranks) { return (int32_t)(((int64_t)r * nparts + nranks - 1) / nranks); }

// Returns false when peer windows are unavailable (the caller falls back to sb_hash_partition + sb_all_to_all).
static bool shuffle_exchange_impl(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t nparts, cudaStream_t st, sb_table **out,
                                  int64_t *out_part_offsets_host) {
  const CommInfo ci = comm_info();
  const int R = ci.nranks, me = ci.rank;
  SB_REQUIRE(ci.up, "sb_shuffle_exchange needs an initialised communicator (sb_comm_init)");
  SB_REQUIRE(R <= REMOTE_MAX_BUCKETS, "the fused exchange supports up to %d ranks", REMOTE_MAX_BUCKETS);
  SB_REQUIRE(nparts >= 1 && nparts <= MULTISPLIT_MAX_BUCKETS, "num_partitions out of range");
  const int64_t n = in->nrows;
  SB_REQUIRE(n < 0xFFFFFFFFll, "tables of 2^32 rows or more must be exchanged in chunks");
  for (auto &c : in->cols)
    if (c.type == SB_STRING) fail(SB_ERR_UNSUPPORTED, "the fused exchange moves fixed-width columns (string columns: sb_hash_partition + sb_all_to_all)");
  OwnerBounds ob;
  for (int r = 0; r <= R; r++) ob.first[r] = owner_first(r, nparts, R);
  // 1. partition ids, destination ranks, per-tile histogram over the ranks
  KeyCols keys = make_keys(in, key_cols, nkeys);
  int64_t rowbytes = 4;
  for (auto &c : in->cols) rowbytes += type_width(c.type);
  const PartGeometry g = part_geometry(n, R, rowbytes >= 32);
  Scratch pid(n * 4 + 16, st), dest(n * 4 + 16, st), hist((int64_t)R * g.nblocks * 4 + 16, st), offs_dev((R + 1) * 8, st);
  if (n > 0) {
    const PartGeometry gp = part_geometry(n, nparts);
    pid_hist_kernel<<<gp.nblocks, PART_THREADS, 0, st>>>(keys, n, nparts, gp.chunk, pid.as<int32_t>(), nullptr, 0, 0);
    SB_LAUNCH_CHECK();
    owner_hist_kernel<<<g.nblocks, PDH_THREADS, 0, st>>>(pid.as<int32_t>(), n, ob, R, g.chunk, dest.as<int32_t>(), hist.as<uint32_t>());
    SB_LAUNCH_CHECK();
  } else SB_CUDA(cudaMemsetAsync(hist.ptr, 0, (size_t)R * g.nblocks * 4, st));
  exclusive_scan_i32((const int32_t *)hist.ptr, (int32_t *)hist.ptr, (int64_t)R * g.nblocks, nullptr, st);
  part_offsets_kernel<<<(R + 1 + 255) / 256, 256, 0, st>>>(hist.as<uint32_t>(), R, g.nblocks, n, offs_dev.as<int64_t>());
  SB_LAUNCH_CHECK();
  std::vector<int64_t> lstart(R + 1);
  SB_CUDA(cudaMemcpyAsync(lstart.data(), offs_dev.ptr, (size_t)(R + 1) * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  // 2. everybody learns everybody's send counts: C[src][dst].  A rank whose column carries no bitmap still has to agree on the
  //    layout, so "nullable" is decided over all ranks (bit mask in the last word, like sb_all_to_all)
  SB_REQUIRE(in->cols.size() <= 62, "the exchange supports up to 62 columns");
  std::vector<int64_t> mine(R + 1), all((size_t)R * (R + 1));
  for (int d = 0; d < R; d++) mine[d] = lstart[d + 1] - lstart[d];
  uint64_t my_mask = 0;
  for (size_t ci2 = 0; ci2 < in->cols.size(); ci2++)
    if (in->cols[ci2].validity) my_mask |= 1ull << ci2;
  mine[R] = (int64_t)my_mask;
  comm_allgather_host(mine.data(), R + 1, all.data(), st);
  uint64_t any_mask = 0;
  for (int r = 0; r < R; r++) any_mask |= (uint64_t)all[(size_t)r * (R + 1) + R];
  auto C = [&](int src, int dst) { return all[(size_t)src * (R + 1) + dst]; };
  std::vector<int64_t> T(R, 0);
  for (int d = 0; d < R; d++)
    for (int sr = 0; sr < R; sr++) T[d] += C(sr, d);
  // 3. window layout of a receiver holding `rows` rows: data columns, the partition-id column, one validity byte column per
  //    nullable column; every piece 256-byte aligned
  struct Piece { int width; const void *src; int col; bool is_valid; };
  std::vector<Piece> pieces;
  std::vector<std::unique_ptr<Scratch>> temps;
  for (size_t i = 0; i < in->cols.size(); i++) pieces.push_back({type_width(in->cols[i].type), in->cols[i].d(), (int)i, false});
  pieces.push_back({4, pid.ptr, -1, false});
  for (size_t i = 0; i < in->cols.size(); i++)
    if ((any_mask >> i) & 1) {
      Scratch *vb = new Scratch(n + 16, st);
      temps.emplace_back(vb);
      bitmap_to_bytes(in->cols[i].v(), n, vb->as<uint8_t>(), st);   // no bitmap on this rank: all ones
      pieces.push_back({1, vb->ptr, (int)i, true});
    }
  auto layout = [&](int64_t rows, std::vector<size_t> &off) {
    size_t cur = 0;
    off.resize(pieces.size());
    for (size_t k = 0; k < pieces.size(); k++) {
      off[k] = cur;
      cur += ((size_t)rows * pieces[k].width + 255) / 256 * 256;
    }
    return cur;
  };
  size_t need = 0;
  std::vector<std::vector<size_t>> offs_of(R);
  for (int d = 0; d < R; d++) need = std::max(need, layout(T[d], offs_of[d]));
  std::vector<void *> bases;
  if (!comm_window(need, st, bases)) return false;
  // 4. the scatter: every destination's run is stored straight into that rank's window (remote stores over NVLink); rows from
  //    source rank s occupy [roff, roff + C[s][d]) of every piece, in arrival order
  if (n > 0) {
    const bool big = g.chunk == RG_TILE_BIG;
    static std::once_flag once;
    std::call_once(once, [] {
      SB_CUDA(cudaFuncSetAttribute(regroup_tma_kernel<512, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RGT_STAGES * RG_TILE_SMALL * 8));
      SB_CUDA(cudaFuncSetAttribute(regroup_tma_kernel<1024, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RGT_STAGES * RG_TILE_BIG * 8));
    });
    const int bps = big ? 1 : 2;
    const int grid = g.nblocks < rt().num_sms * bps ? g.nblocks : rt().num_sms * bps;
    KernelTimer kt("exchange_scatter", st);
    for (size_t done = 0; done < pieces.size();) {
      RegroupCols rc;
      memset(&rc, 0, sizeof(rc));
      std::vector<uint64_t> hp;
      while (done < pieces.size() && rc.ncols < SCATTER_MAX_COLS) {
        const Piece &pc = pieces[done];
        const int k = rc.ncols++;
        rc.width[k] = pc.width;
        rc.src[k] = pc.src;
        for (int d = 0; d < R; d++) {
          int64_t roff = 0;
          for (int sr = 0; sr < me; sr++) roff += C(sr, d);
          // biased so that global sorted position g of the LOCAL bucket order lands at window position roff + (g - lstart[d])
          const intptr_t addr = (intptr_t)bases[d] + (intptr_t)offs_of[d][done] + (intptr_t)(roff - lstart[d]) * pc.width;
          hp.push_back((uint64_t)addr);
        }
        done++;
      }
      Scratch *dp = new Scratch((int64_t)hp.size() * 8 + 8, st);
      temps.emplace_back(dp);
      SB_CUDA(cudaMemcpyAsync(dp->ptr, hp.data(), hp.size() * 8, cudaMemcpyHostToDevice, st));
      SB_CUDA(cudaStreamSynchronize(st));   // hp is a temporary
      if (big)
        regroup_tma_kernel<1024, true><<<grid, 1024, RGT_STAGES * RG_TILE_BIG * 8, st>>>(rc, dest.as<int32_t>(), hist.as<uint32_t>(), n, R, (int64_t)g.nblocks,
                                                                                         nullptr, 0, dp->as<uint64_t>());
      else
        regroup_tma_kernel<512, true><<<grid, 512, RGT_STAGES * RG_TILE_SMALL * 8, st>>>(rc, dest.as<int32_t>(), hist.as<uint32_t>(), n, R, (int64_t)g.nblocks,
                                                                                        nullptr, 0, dp->as<uint64_t>());
      SB_LAUNCH_CHECK();
    }
  }
  // 5. every rank's stores have landed once every rank has passed this point on its stream
  comm_barrier_enqueue(st);
  // 6. receiver side: split the window's rows (grouped by source rank) into the owned partitions -- the second, local pass
  const int64_t nrecv = T[me];
  const int32_t lo = ob.first[me], hi = ob.first[me + 1], nb2 = hi - lo;
  const uint8_t *win = (const uint8_t *)bases[me];
  const std::vector<size_t> &woff = offs_of[me];
  sb_table *t = table_new(nrecv);
  try {
    std::vector<SplitCol> sc;
    std::vector<std::pair<size_t, Scratch *>> vbytes;   // (column, received validity bytes in output order)
    for (size_t i = 0; i < in->cols.size(); i++) {
      const Column &c = in->cols[i];
      Column r = column_alloc(c.type, c.scale, nrecv, ((any_mask >> i) & 1) != 0, st);
      t->cols.push_back(r);
      sc.push_back({type_width(c.type), win + woff[i], r.data->ptr, nullptr, nullptr});
    }
    const size_t pid_piece = in->cols.size();
    for (size_t k = pid_piece + 1; k < pieces.size(); k++) {
      Scratch *vb = new Scratch(nrecv + 16, st);
      temps.emplace_back(vb);
      vbytes.push_back({(size_t)pieces[k].col, vb});
      sc.push_back({1, win + woff[k], vb->ptr, nullptr, nullptr});
    }
    std::vector<int64_t> offs2((size_t)std::max(nb2, 1) + 1, 0);
    if (nrecv > 0 && nb2 > 0) {
      const PartGeometry g2 = part_geometry(nrecv, nb2, rowbytes >= 32 && nb2 >= 64);
      Scratch bucket2(nrecv * 4 + 16, st), hist2((int64_t)nb2 * g2.nblocks * 4 + 16, st), offs2_dev((int64_t)(nb2 + 1) * 8, st);
      static bool attr = false;
      if (!attr) {
        SB_CUDA(cudaFuncSetAttribute(local_pid_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
        attr = true;
      }
      local_pid_hist_kernel<<<g2.nblocks, PDH_THREADS, (size_t)nb2 * 4, st>>>((const int32_t *)(win + woff[pid_piece]), nrecv, lo, nb2, g2.chunk,
                                                                            bucket2.as<int32_t>(), hist2.as<uint32_t>());
      SB_LAUNCH_CHECK();
      multisplit_scatter(bucket2.as<int32_t>(), hist2.as<uint32_t>(), nb2, g2, sc.data(), (int)sc.size(), nrecv, nullptr, offs2_dev.as<int64_t>(), st);
      SB_CUDA(cudaMemcpyAsync(offs2.data(), offs2_dev.ptr, (size_t)(nb2 + 1) * 8, cudaMemcpyDeviceToHost, st));
    }
    for (auto &vb : vbytes) bytes_to_bitmap(vb.second->as<uint8_t>(), nrecv, (uint32_t *)t->cols[vb.first].validity->ptr, st);
    SB_CUDA(cudaStreamSynchronize(st));
    out_part_offsets_host[0] = 0;
    for (int p = 0; p < nparts; p++) {
      const int64_t rows = (p >= lo && p < hi) ? offs2[p - lo + 1] - offs2[p - lo] : 0;
      out_part_offsets_host[p + 1] = out_part_offsets_host[p] + rows;
    }
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
  return true;
}

}  // namespace sb

using namespace sb;

extern "C" {

int sb_partition_ids(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t num_partitions, sb_stream *s,
                     int32_t *out_ids_device) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(in && out_ids_device, "null argument");
  SB_REQUIRE(num_partitions >= 1, "num_partitions must be >= 1");
  cudaStream_t st = stream_of(s);
  KeyCols keys = make_keys(in, key_cols, nkeys);
  int64_t n = in->nrows;
  if (n > 0) {
    PartGeometry g = part_geometry(n, num_partitions);
    pid_hist_kernel<<<g.nblocks, PART_THREADS, 0, st>>>(keys, n, num_partitions, g.chunk, out_ids_device, nullptr, 0, 0);
    SB_LAUNCH_CHECK();
  }
  SB_API_END
}

int sb_hash_partition(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t num_partitions, sb_stream *s,
                      sb_table **out, int64_t *out_offsets_host) {
  SB_API_BEGIN
  require_init();
  partition_impl(in, key_cols, nkeys, num_partitions, 0, 0, stream_of(s), out, out_offsets_host);
  SB_API_END
}

// ShuffleExchangeExec with HashPartitioning in ONE call: map side and transport fused (see shuffle_exchange_impl).  Falls back to
// sb_hash_partition + sb_all_to_all when peer windows cannot be mapped.
int sb_shuffle_exchange(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t num_partitions, sb_stream *s, sb_table **out,
                        int64_t *out_part_offsets_host) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(in && out && out_part_offsets_host, "null argument");
  bool has_string = false;
  for (auto &c : in->cols) has_string |= c.type == SB_STRING || c.type == SB_DECIMAL128;   // not moved by the fused kernels
  if (!has_string && !config().exchange_nccl && shuffle_exchange_impl(in, key_cols, nkeys, num_partitions, stream_of(s), out, out_part_offsets_host))
    return SB_OK;
  sb_table *parted = nullptr;
  std::vector<int64_t> offs((size_t)num_partitions + 1);
  partition_impl(in, key_cols, nkeys, num_partitions, 0, 0, stream_of(s), &parted, offs.data());
  const int rc = sb_all_to_all(parted, offs.data(), num_partitions, s, out, out_part_offsets_host);
  sb_table_release(parted);
  if (rc != SB_OK) return rc;
  SB_API_END
}

int sb_round_robin_partition(const sb_table *in, int32_t start, int32_t num_partitions, sb_stream *s, sb_table **out,
                             int64_t *out_offsets_host) {
  SB_API_BEGIN
  require_init();
  partition_impl(in, nullptr, 0, num_partitions, 1, start, stream_of(s), out, out_offsets_host);
  SB_API_END
}

}  // extern "C"
