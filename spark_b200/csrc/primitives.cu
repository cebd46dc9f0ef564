// primitives.cu -- exclusive scan, gather, compaction.
#include "primitives.cuh"

namespace sb {

// ------------------------------------------------------------------------------------ scan
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T *smem_warp /* 32 */, T &block_total) {
  // inclusive warp scan
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    T y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) smem_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    T w = lane < (blockDim.x >> 5) ? smem_warp[lane] : (T)0;
    T s = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      T y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    smem_warp[lane] = s - w;  // exclusive warp offsets; total = last inclusive
    if (lane == 31) smem_warp[32] = s;
  }
  __syncthreads();
  T res = smem_warp[warp] + x - v;
  block_total = smem_warp[32];
  return res;
}

template <typename Tin, typename Tout>
__global__ void __launch_bounds__(SCAN_THREADS) scan_reduce_kernel(const Tin *__restrict__ in, Tout *__restrict__ partials, int64_t n) {
  __shared__ Tout sm[33];
  int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
  Tout s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++)
    if (base + k < n) s += (Tout)in[base + k];
  Tout tot;
  block_exclusive_scan<Tout>(s, sm, tot);
  if (threadIdx.x == 0) partials[blockIdx.x] = tot;
}

template <typename Tin, typename Tout>
__global__ void __launch_bounds__(SCAN_THREADS) scan_down_kernel(const Tin *in, Tout *out, const Tout *__restrict__ partials_excl,
                                                                 int64_t n, Tout *total) {
  __shared__ Tout sm[33];
  int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
  Tout v[SCAN_ITEMS];
  Tout s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    v[k] = base + k < n ? (Tout)in[base + k] : (Tout)0;
    s += v[k];
  }
  Tout tot;
  Tout ex = block_exclusive_scan<Tout>(s, sm, tot);
  Tout off = (partials_excl ? partials_excl[blockIdx.x] : (Tout)0) + ex;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    if (base + k < n) out[base + k] = off;
    off += v[k];
  }
  if (total && blockIdx.x == gridDim.x - 1 && threadIdx.x == SCAN_THREADS - 1) *total = off;
}

template <typename Tin, typename Tout>
static void exclusive_scan_impl(const Tin *in, Tout *out, int64_t n, Tout *total_dev, cudaStream_t st) {
  if (n <= 0) {
    if (total_dev) SB_CUDA(cudaMemsetAsync(total_dev, 0, sizeof(Tout), st));
    return;
  }
  int64_t nb = (n + SCAN_TILE - 1) / SCAN_TILE;
  if (nb == 1) {
    scan_down_kernel<Tin, Tout><<<1, SCAN_THREADS, 0, st>>>(in, out, nullptr, n, total_dev);
    SB_LAUNCH_CHECK();
    return;
  }
  Scratch partials(sizeof(Tout) * nb, st);
  scan_reduce_kernel<Tin, Tout><<<(unsigned)nb, SCAN_THREADS, 0, st>>>(in, partials.as<Tout>(), n);
  SB_LAUNCH_CHECK();
  exclusive_scan_impl<Tout, Tout>(partials.as<Tout>(), partials.as<Tout>(), nb, nullptr, st);
  scan_down_kernel<Tin, Tout><<<(unsigned)nb, SCAN_THREADS, 0, st>>>(in, out, partials.as<Tout>(), n, total_dev);
  SB_LAUNCH_CHECK();
}

void exclusive_scan_i64(const int64_t *in, int64_t *out, int64_t n, int64_t *total_dev, cudaStream_t st) {
  exclusive_scan_impl<int64_t, int64_t>(in, out, n, total_dev, st);
}
void exclusive_scan_i32(const int32_t *in, int32_t *out, int64_t n, int32_t *total_dev, cudaStream_t st) {
  exclusive_scan_impl<int32_t, int32_t>(in, out, n, total_dev, st);
}
void exclusive_scan_i32_to_i64(const int32_t *in, int64_t *out, int64_t n, int64_t *total_dev, cudaStream_t st) {
  exclusive_scan_impl<int32_t, int64_t>(in, out, n, total_dev, st);
}

// ------------------------------------------------------------------------------------ gather
constexpr int GATHER_MAX_COLS = 12;
static inline unsigned gather_grid(int64_t nout) { return (unsigned)((nout + 256 * 8 - 1) / (256 * 8)); }
struct GatherArgs {
  int ncols;
  int width[GATHER_MAX_COLS];
  const void *src[GATHER_MAX_COLS];
  void *dst[GATHER_MAX_COLS];
  const uint8_t *src_valid[GATHER_MAX_COLS];
  uint32_t *dst_valid[GATHER_MAX_COLS];   // null -> no validity output
};

// A thread owns GATHER_ITEMS rows (block-strided, so every index load and every store is a coalesced sweep) and, column by column, issues
// the loads of all its rows before the first store: a row gather is latency-bound (one 32-byte sector per value), what matters is how many
// sectors are in flight.  (One row per thread with the column loop not unrolled kept one load in flight per thread.)
constexpr int GATHER_ITEMS = 8;
template <typename T>
__device__ __forceinline__ void gather_rows(const void *__restrict__ src, void *__restrict__ dst, const int64_t (&j)[GATHER_ITEMS], int64_t i0, int64_t nout) {
  T v[GATHER_ITEMS];
#pragma unroll
  for (int k = 0; k < GATHER_ITEMS; k++) v[k] = j[k] >= 0 ? __ldg((const T *)src + j[k]) : T{};
#pragma unroll
  for (int k = 0; k < GATHER_ITEMS; k++)
    if (i0 + k * 256 < nout) ((T *)dst)[i0 + k * 256] = v[k];
}
template <bool ALIGNED16>
__device__ __forceinline__ void gather_rows16(const void *__restrict__ src, void *__restrict__ dst, const int64_t (&j)[GATHER_ITEMS], int64_t i0,
                                              int64_t nout) {
#pragma unroll
  for (int h = 0; h < 2; h++) {   // two halves: 16-byte values would double the register footprint
    uint4 v[GATHER_ITEMS / 2];
#pragma unroll
    for (int k = 0; k < GATHER_ITEMS / 2; k++) {
      const int64_t jj = j[h * (GATHER_ITEMS / 2) + k];
      if (jj < 0) {
        v[k] = make_uint4(0, 0, 0, 0);
      } else if (ALIGNED16) {
        v[k] = __ldg((const uint4 *)src + jj);
      } else {
        const uint2 lo = __ldg((const uint2 *)src + 2 * jj), hi = __ldg((const uint2 *)src + 2 * jj + 1);
        v[k] = make_uint4(lo.x, lo.y, hi.x, hi.y);
      }
    }
#pragma unroll
    for (int k = 0; k < GATHER_ITEMS / 2; k++) {
      const int64_t i = i0 + (h * (GATHER_ITEMS / 2) + k) * 256;
      if (i < nout) ((uint4 *)dst)[i] = v[k];
    }
  }
}
__global__ void __launch_bounds__(256) gather_fixed_kernel(GatherArgs a, const int64_t *__restrict__ idx, int64_t nout) {
  const int64_t i0 = (int64_t)blockIdx.x * (256 * GATHER_ITEMS) + threadIdx.x;
  int64_t j[GATHER_ITEMS];
#pragma unroll
  for (int k = 0; k < GATHER_ITEMS; k++) j[k] = i0 + k * 256 < nout ? idx[i0 + k * 256] : -1;
#pragma unroll 1
  for (int c = 0; c < a.ncols; c++) {
    switch (a.width[c]) {
      case 1: gather_rows<uint8_t>(a.src[c], a.dst[c], j, i0, nout); break;
      case 2: gather_rows<uint16_t>(a.src[c], a.dst[c], j, i0, nout); break;
      case 4: gather_rows<uint32_t>(a.src[c], a.dst[c], j, i0, nout); break;
      case 16:
        // a 16-byte load needs a 16-byte aligned source; a decimal128 column borrowed from device memory may be only 8-byte
        // aligned (test_gpu_row_movement.py::test_shuffle_misaligned_source faulted on it), and then takes two 8-byte loads
        if (((uintptr_t)a.src[c] & 15) == 0) gather_rows16<true>(a.src[c], a.dst[c], j, i0, nout);
        else gather_rows16<false>(a.src[c], a.dst[c], j, i0, nout);
        break;
      default: gather_rows<uint64_t>(a.src[c], a.dst[c], j, i0, nout); break;
    }
    if (a.dst_valid[c]) {
      const uint8_t *sv = a.src_valid[c];
      bool v[GATHER_ITEMS];
      if (sv) {
        uint8_t b[GATHER_ITEMS];
#pragma unroll
        for (int k = 0; k < GATHER_ITEMS; k++) b[k] = j[k] >= 0 ? __ldg(sv + (j[k] >> 3)) : 0;
#pragma unroll
        for (int k = 0; k < GATHER_ITEMS; k++) v[k] = j[k] >= 0 && ((b[k] >> (j[k] & 7)) & 1);
      } else {
#pragma unroll
        for (int k = 0; k < GATHER_ITEMS; k++) v[k] = j[k] >= 0;
      }
#pragma unroll
      for (int k = 0; k < GATHER_ITEMS; k++) {
        const uint32_t word = __ballot_sync(0xffffffffu, v[k]);
        const int64_t i = i0 + k * 256;
        if ((threadIdx.x & 31) == 0 && i < nout) a.dst_valid[c][i >> 5] = word;
      }
    }
  }
}

// strings: lengths -> scan -> byte copy (one warp per row)
__global__ void gather_str_len_kernel(const int32_t *__restrict__ src_off, const int64_t *__restrict__ idx, int64_t nout,
                                      int32_t *__restrict__ out_len) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nout) return;
  int64_t j = idx[i];
  out_len[i] = j >= 0 ? src_off[j + 1] - src_off[j] : 0;
}
__global__ void gather_str_copy_kernel(const uint8_t *__restrict__ src, const int32_t *__restrict__ src_off,
                                       const int64_t *__restrict__ idx, int64_t nout, const int32_t *__restrict__ dst_off,
                                       uint8_t *__restrict__ dst) {
  int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (w >= nout) return;
  int64_t j = idx[w];
  if (j < 0) return;
  int32_t so = src_off[j], len = src_off[j + 1] - so, d = dst_off[w];
  for (int k = lane; k < len; k += 32) dst[d + k] = src[so + k];
}

static Column gather_string(const Column &c, const int64_t *idx, int64_t nout, bool neg, cudaStream_t st) {
  Column r;
  r.type = c.type;
  r.length = nout;
  r.offsets = buffer_alloc((nout + 1) * 4 + 16, st);
  int32_t *off = (int32_t *)r.offsets->ptr;
  Scratch total(8, st);
  if (nout > 0) {
    gather_str_len_kernel<<<(unsigned)((nout + 255) / 256), 256, 0, st>>>(c.o(), idx, nout, off);
    SB_LAUNCH_CHECK();
  }
  // scan over nout lengths, writing nout+1 offsets: scan in place then append the total
  exclusive_scan_i32(off, off, nout, total.as<int32_t>(), st);
  SB_CUDA(cudaMemcpyAsync(off + nout, total.ptr, 4, cudaMemcpyDeviceToDevice, st));
  int32_t bytes = 0;
  SB_CUDA(cudaMemcpyAsync(&bytes, total.ptr, 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  r.string_bytes = bytes;
  r.data = buffer_alloc(bytes + 16, st);
  if (nout > 0 && bytes > 0) {
    gather_str_copy_kernel<<<(unsigned)((nout * 32 + 255) / 256), 256, 0, st>>>((const uint8_t *)c.d(), c.o(), idx, nout, off,
                                                                               (uint8_t *)r.data->ptr);
    SB_LAUNCH_CHECK();
  }
  if (c.validity || neg) {
    r.validity = buffer_alloc(bitmap_alloc_bytes(nout), st);
    r.null_count = -1;
    GatherArgs a;
    a.ncols = 1;
    a.width[0] = 0;   // validity only: width 0 hits the default store... avoid: handled below
    a.src[0] = nullptr;
    a.dst[0] = nullptr;
    a.src_valid[0] = c.v();
    a.dst_valid[0] = (uint32_t *)r.validity->ptr;
    // reuse the fixed kernel with a dummy 1-byte column
    Scratch dummy_src(16, st), dummy_dst(nout + 16, st);
    (void)dummy_src;
    a.width[0] = 1;
    a.dst[0] = dummy_dst.ptr;
    a.src[0] = c.d();
    if (nout > 0) {
      // src[j] read of 1 byte must be in-bounds: use the offsets buffer (>= 4*(n+1) bytes) instead
      a.src[0] = c.o();
      gather_fixed_kernel<<<gather_grid(nout), 256, 0, st>>>(a, idx, nout);
      SB_LAUNCH_CHECK();
    }
  }
  return r;
}

Column gather_column(const Column &c, const int64_t *idx, int64_t nout, bool neg, cudaStream_t st) {
  if (c.type == SB_STRING) return gather_string(c, idx, nout, neg, st);
  Column r = column_alloc(c.type, c.scale, nout, c.validity != nullptr || neg, st);
  if (nout == 0) return r;
  GatherArgs a;
  a.ncols = 1;
  a.width[0] = type_width(c.type);
  a.src[0] = c.d();
  a.dst[0] = r.data->ptr;
  a.src_valid[0] = c.v();
  a.dst_valid[0] = r.validity ? (uint32_t *)r.validity->ptr : nullptr;
  gather_fixed_kernel<<<gather_grid(nout), 256, 0, st>>>(a, idx, nout);
  SB_LAUNCH_CHECK();
  return r;
}

sb_table *gather_table(const sb_table *in, const int64_t *idx, int64_t nout, bool neg, cudaStream_t st, int skip_col) {
  KernelTimer kt("gather", st);
  sb_table *t = table_new(nout);
  try {
    t->cols.resize(in->cols.size());
    GatherArgs a;
    a.ncols = 0;
    auto flush = [&]() {
      if (a.ncols && nout > 0) {
        gather_fixed_kernel<<<gather_grid(nout), 256, 0, st>>>(a, idx, nout);
        SB_LAUNCH_CHECK();
      }
      a.ncols = 0;
    };
    for (size_t i = 0; i < in->cols.size(); i++) {
      const Column &c = in->cols[i];
      if ((int)i == skip_col) continue;
      if (c.type == SB_STRING) {
        t->cols[i] = gather_string(c, idx, nout, neg, st);
        continue;
      }
      Column r = column_alloc(c.type, c.scale, nout, c.validity != nullptr || neg, st);
      t->cols[i] = r;
      int k = a.ncols++;
      a.width[k] = type_width(c.type);
      a.src[k] = c.d();
      a.dst[k] = r.data->ptr;
      a.src_valid[k] = c.v();
      a.dst_valid[k] = r.validity ? (uint32_t *)r.validity->ptr : nullptr;
      if (a.ncols == GATHER_MAX_COLS) flush();
    }
    flush();
  } catch (...) {
    table_free(t);
    throw;
  }
  return t;
}

// ------------------------------------------------------------------------------------ compaction
// Two passes over the mask (1 B/row each) instead of mask -> int32 flags -> scan -> int64 positions -> write (25 B/row):
// pass 1 counts the survivors of every 4096-row tile, a tiny scan turns the counts into tile offsets, pass 2 re-reads the
// tile, ranks the survivors inside the block (thread-local count, warp shuffle scan, 8 warp totals) and writes their row ids.
constexpr int CM_THREADS = 256;
constexpr int CM_ITEMS = 16;                       // consecutive rows per thread: one 16-byte load
constexpr int CM_TILE = CM_THREADS * CM_ITEMS;     // 4096 rows

__device__ __forceinline__ uint32_t cm_load_bits(const uint8_t *__restrict__ mask, int64_t row0, int64_t n, bool aligned) {
  uint32_t bits = 0;
  if (aligned && row0 + CM_ITEMS <= n) {
    const uint4 v = *reinterpret_cast<const uint4 *>(mask + row0);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int b = 0; b < 4; b++) bits |= ((w[j] >> (8 * b)) & 0xFFu) ? 1u << (4 * j + b) : 0u;
  } else {
#pragma unroll
    for (int j = 0; j < CM_ITEMS; j++)
      if (row0 + j < n && mask[row0 + j]) bits |= 1u << j;
  }
  return bits;
}

__global__ void __launch_bounds__(CM_THREADS) compact_count_kernel(const uint8_t *__restrict__ mask, int64_t n, bool aligned,
                                                                   int32_t *__restrict__ tile_counts) {
  __shared__ int32_t wsum[CM_THREADS / 32];
  const int64_t row0 = (int64_t)blockIdx.x * CM_TILE + (int64_t)threadIdx.x * CM_ITEMS;
  int32_t c = __popc(cm_load_bits(mask, row0, n, aligned));
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t t = 0;
#pragma unroll
    for (int w = 0; w < CM_THREADS / 32; w++) t += wsum[w];
    tile_counts[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(CM_THREADS) compact_write_kernel(const uint8_t *__restrict__ mask, int64_t n, bool aligned,
                                                                   const int64_t *__restrict__ tile_offsets, int64_t *__restrict__ out) {
  __shared__ int32_t wsum[CM_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * CM_TILE + (int64_t)threadIdx.x * CM_ITEMS;
  uint32_t bits = cm_load_bits(mask, row0, n, aligned);
  const int32_t c = __popc(bits);
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
  int64_t *dst = out + tile_offsets[blockIdx.x] + woff + (x - c);
  while (bits) {
    const int j = __ffs(bits) - 1;
    bits &= bits - 1;
    *dst++ = row0 + j;
  }
}

void compact_mask_async(const uint8_t *mask, int64_t n, int64_t *out_idx, int32_t *tile_counts, int64_t *tile_offsets, int64_t *total_dev,
                        cudaStream_t st) {
  if (n == 0) {
    SB_CUDA(cudaMemsetAsync(total_dev, 0, 8, st));
    return;
  }
  const unsigned nb = (unsigned)compact_tiles(n);
  const bool aligned = ((uintptr_t)mask & 15) == 0;
  compact_count_kernel<<<nb, CM_THREADS, 0, st>>>(mask, n, aligned, tile_counts);
  SB_LAUNCH_CHECK();
  exclusive_scan_i32_to_i64(tile_counts, tile_offsets, nb, total_dev, st);
  compact_write_kernel<<<nb, CM_THREADS, 0, st>>>(mask, n, aligned, tile_offsets, out_idx);
  SB_LAUNCH_CHECK();
}

int64_t compact_mask(const uint8_t *mask, int64_t n, int64_t *out_idx, cudaStream_t st) {
  if (n == 0) return 0;
  const int64_t nb = compact_tiles(n);
  Scratch counts(nb * 4 + 16, st), offsets(nb * 8 + 16, st), total(8, st);
  compact_mask_async(mask, n, out_idx, counts.as<int32_t>(), offsets.as<int64_t>(), total.as<int64_t>(), st);
  int64_t cnt = 0;
  SB_CUDA(cudaMemcpyAsync(&cnt, total.ptr, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return cnt;
}

__global__ void bitmap_to_bytes_kernel(const uint8_t *__restrict__ bm, int64_t n, uint8_t *__restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = bit_valid(bm, i) ? 1 : 0;
}
__global__ void bytes_to_bitmap_kernel(const uint8_t *__restrict__ in, int64_t n, uint32_t *__restrict__ bm) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool v = i < n && in[i];
  uint32_t w = __ballot_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && (i - (i & 31)) < n) bm[i >> 5] = w;
}
void bitmap_to_bytes(const uint8_t *bm, int64_t n, uint8_t *out, cudaStream_t st) {
  if (n <= 0) return;
  bitmap_to_bytes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(bm, n, out);
  SB_LAUNCH_CHECK();
}
void bytes_to_bitmap(const uint8_t *in, int64_t n, uint32_t *bm, cudaStream_t st) {
  if (n <= 0) return;
  bytes_to_bitmap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, n, bm);
  SB_LAUNCH_CHECK();
}

// string concat: offsets of one piece rebased onto the concatenated character buffer
__global__ void rebase_offsets_kernel(const int32_t *__restrict__ in, int64_t n, int32_t char_base, int32_t *__restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i] - in[0] + char_base;
}

__global__ void iota_kernel(int64_t *out, int64_t n, int64_t begin) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = begin + i;
}
void iota_i64(int64_t *out, int64_t n, int64_t begin, cudaStream_t st) {
  if (n <= 0) return;
  iota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out, n, begin);
  SB_LAUNCH_CHECK();
}

}  // namespace sb

using namespace sb;

extern "C" {

int sb_table_slice(const sb_table *t, int64_t begin, int64_t end, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(t && out && begin >= 0 && end >= begin && end <= t->nrows, "slice [%lld,%lld) out of range", (long long)begin,
             (long long)end);
  cudaStream_t st = stream_of(s);
  int64_t n = end - begin;
  Scratch idx(n * 8 + 8, st);
  iota_i64(idx.as<int64_t>(), n, begin, st);
  *out = gather_table(t, idx.as<int64_t>(), n, false, st);
  SB_API_END
}

int sb_table_concat(const sb_table *const *tables, int32_t ntables, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(tables && ntables >= 1 && out, "concat needs at least one table");
  cudaStream_t st = stream_of(s);
  const sb_table *first = tables[0];
  int64_t total = 0;
  for (int i = 0; i < ntables; i++) {
    SB_REQUIRE(tables[i]->cols.size() == first->cols.size(), "concat: schema mismatch");
    total += tables[i]->nrows;
  }
  sb_table *r = table_new(total);
  try {
    for (size_t c = 0; c < first->cols.size(); c++) {
      int32_t type = first->cols[c].type;
      bool any_valid = false;
      int64_t chars = 0;
      for (int i = 0; i < ntables; i++) {
        SB_REQUIRE(tables[i]->cols[c].type == type, "concat: column %zu type mismatch", c);
        any_valid |= tables[i]->cols[c].validity != nullptr;
        chars += tables[i]->cols[c].string_bytes;
      }
      if (type == SB_STRING) {
        SB_REQUIRE(chars <= INT32_MAX, "concat: string column %zu would exceed 2 GiB of characters", c);
        Column col;
        col.type = SB_STRING;
        col.length = total;
        col.string_bytes = chars;
        col.offsets = buffer_alloc((total + 1) * 4 + 16, st);
        col.data = buffer_alloc(chars + 16, st);
        r->cols.push_back(col);
        int64_t off = 0, cbase = 0;
        for (int i = 0; i < ntables; i++) {
          const Column &pc = tables[i]->cols[c];
          int64_t n = tables[i]->nrows;
          if (n) {
            rebase_offsets_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pc.o(), n, (int32_t)cbase, (int32_t *)col.offsets->ptr + off);
            SB_LAUNCH_CHECK();
          }
          if (pc.string_bytes)
            SB_CUDA(cudaMemcpyAsync((char *)col.data->ptr + cbase, pc.d(), (size_t)pc.string_bytes, cudaMemcpyDeviceToDevice, st));
          off += n;
          cbase += pc.string_bytes;
        }
        int32_t last = (int32_t)chars;
        SB_CUDA(cudaMemcpyAsync((int32_t *)col.offsets->ptr + total, &last, 4, cudaMemcpyHostToDevice, st));
        SB_CUDA(cudaStreamSynchronize(st));   // `last` lives on this frame
      } else {
        int w = type_width(type);
        Column col = column_alloc(type, first->cols[c].scale, total, false, st);
        int64_t off = 0;
        for (int i = 0; i < ntables; i++) {
          int64_t n = tables[i]->nrows;
          if (n) SB_CUDA(cudaMemcpyAsync((char *)col.data->ptr + off * w, tables[i]->cols[c].d(), (size_t)(n * w),
                                         cudaMemcpyDeviceToDevice, st));
          off += n;
        }
        r->cols.push_back(col);
      }
      if (any_valid) {
        // validity: pieces start at arbitrary bit offsets, so go through one byte per row on the device
        Column &rc = r->cols.back();
        rc.validity = buffer_alloc(bitmap_alloc_bytes(total), st);
        rc.null_count = -1;
        Scratch bytes(total + 16, st);
        int64_t o = 0;
        for (int i = 0; i < ntables; i++) {
          int64_t n = tables[i]->nrows;
          bitmap_to_bytes(tables[i]->cols[c].v(), n, bytes.as<uint8_t>() + o, st);
          o += n;
        }
        bytes_to_bitmap(bytes.as<uint8_t>(), total, (uint32_t *)rc.validity->ptr, st);
      }
    }
  } catch (...) {
    table_free(r);
    throw;
  }
  *out = r;
  SB_API_END
}

}  // extern "C"
