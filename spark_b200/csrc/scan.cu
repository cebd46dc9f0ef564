// scan.cu -- the columnar scan boundary: Parquet column-chunk pages (host memory) -> Arrow columns in HBM.
//
// Reference path replaced (SQLJ = sql/core/src/main/java/org/apache/spark/sql/execution/datasources/parquet):
//   FileSourceScanExec.doExecuteColumnar (SQLX/DataSourceScanExec.scala:735-760) pulls ColumnarBatches from
//   VectorizedParquetRecordReader.nextBatch (SQLJ/VectorizedParquetRecordReader.java), whose per-column work is
//   VectorizedColumnReader.readBatch (SQLJ/VectorizedColumnReader.java:321-460: readPageV1 / readPageV2, definition levels,
//   initDataReader), VectorizedRleValuesReader (SQLJ/VectorizedRleValuesReader.java:95-117 initFromPage, :981-1020
//   readNextGroup: the RLE / bit-packed hybrid) and VectorizedPlainValuesReader, decoding on the CPU into
//   OffHeapColumnVectors that RowToColumnar / the plugin would then copy to the device.
// Here the ENCODED page bytes cross PCIe (one copy per column chunk) and the GPU decodes them: for TPC-H lineitem the
// dictionary-encoded columns are 1-12 bits per value instead of 8-64, which is what the end-to-end rate is bound by.
//
// Supported: physical types BOOLEAN / INT32 / INT64 / FLOAT / DOUBLE, and BYTE_ARRAY decoded to SB_STRING; encodings PLAIN,
// RLE_DICTIONARY (= PLAIN_DICTIONARY: bit-width byte + hybrid runs over a PLAIN dictionary page), DELTA_BINARY_PACKED (INT32 /
// INT64), DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY (BYTE_ARRAY); data pages V1 (levels length-prefixed in front of the
// values) and V2 (levels in their own section); flat schemas (max definition level <= 1, no repetition); uncompressed pages, or
// SNAPPY pages through sb_scan_decode_compressed (decompressed on the device by snappy.cu).  FIXED_LEN_BYTE_ARRAY, INT96 and
// BYTE_STREAM_SPLIT are rejected with SB_ERR_UNSUPPORTED rather than decoded on the CPU.
//
// Kernel: one 256-thread block per page.  (1) definition levels -> one validity byte per row; (2) values -> dense value
// space (page-local), PLAIN by a widening/narrowing copy, RLE_DICTIONARY by walking the hybrid stream: thread 0 parses up
// to 64 run headers into shared memory, then the whole block decodes those runs' values in parallel (value i of the batch
// finds its run by binary search in the batch's prefix sums -- balanced whatever the run lengths are) and gathers from the
// dictionary; (3) NULLable pages: block scan of the validity bytes maps rows to value indices (out[row] = dense[idx]).
// Algorithmic bytes: encoded bytes read once + decoded column written once.
#include <algorithm>
#include <memory>
#include "common.cuh"
#include "primitives.cuh"
#include "snappy.cuh"

namespace sb {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_RUNS = 64;

struct PageTask {
  const uint8_t *values;     // device: encoded values of the page
  const uint8_t *def;        // device: definition-level hybrid stream (bit width 1) or nullptr
  int64_t values_bytes, def_bytes;
  int64_t row_start;         // first row of the page in the column
  int32_t num_values;        // rows of the page (NULLs included)
  int32_t encoding;          // SB_ENC_*
  int32_t col;
  int32_t pad;
};
struct ColTask {
  void *out;                 // decoded column (row space)
  uint8_t *valid_bytes;      // one byte per row, or nullptr when no page of the column carries definition levels
  uint8_t *dense;            // value-space staging for NULLable columns (same size as out), else nullptr
  const uint8_t *dict;       // device: PLAIN dictionary values
  int32_t dict_count;
  int32_t phys_width;        // 0 BOOLEAN (bit-packed), 4, 8
  int32_t out_width;         // 1, 2, 4, 8
  int32_t mul;               // sb_column_chunk.value_multiplier (<= 1: values as stored)
};

__device__ __forceinline__ uint64_t load_le(const uint8_t *p, int nbytes) {
  uint64_t w = 0;
  for (int b = 0; b < nbytes; b++) w |= (uint64_t)p[b] << (8 * b);
  return w;
}
__device__ __forceinline__ void store_value(void *out, int width, int64_t i, uint64_t v) {
  switch (width) {
    case 1: ((uint8_t *)out)[i] = (uint8_t)v; break;
    case 2: ((uint16_t *)out)[i] = (uint16_t)v; break;
    case 4: ((uint32_t *)out)[i] = (uint32_t)v; break;
    default: ((uint64_t *)out)[i] = v; break;
  }
}

// a physical value as the column holds it: INT32 sign-extended into a decimal64, then the unit multiplier (TIMESTAMP(MILLIS) ->
// microseconds; wraps like the reference's long arithmetic would before its overflow check)
__device__ __forceinline__ uint64_t column_value(uint64_t v, int pw, int ow, int32_t mul) {
  if (pw == 4 && ow == 8) v = (uint64_t)(int64_t)(int32_t)v;   // decimal(p <= 9) stored as INT32
  if (mul > 1) v *= (uint64_t)mul;
  return v;
}

// unsigned LEB128 at p[pos] (bounded by nbytes); returns the value, *len = bytes consumed
__device__ __forceinline__ uint32_t read_uvarint(const uint8_t *__restrict__ p, int64_t pos, int64_t nbytes, int *len) {
  uint32_t v = 0;
  int shift = 0, l = 0;
  while (pos + l < nbytes) {
    const uint8_t b = p[pos + l++];
    v |= (uint32_t)(b & 0x7f) << shift;
    shift += 7;
    if (!(b & 0x80) || shift > 28) break;
  }
  *len = l;
  return v;
}

// Walks an RLE / bit-packed hybrid stream (VectorizedRleValuesReader.readNextGroup) and calls emit(index, value) for the first
// max_values values.  Block-cooperative; returns the number of values produced (same in every thread).
//   * Run headers form a chain (a header says where the next one is), and every link costs a memory round trip.  Writers emit
//     long stretches of identical runs (parquet-mr: bit-packed runs of 504 values, header 0x7F), so warp 0 walks the chain
//     SPECULATIVELY: it reads the header at the cursor, then lane l checks that the same header sits l run-lengths further
//     on; the leading lanes that agree are 32 links resolved in two round trips instead of 32.  Irregular streams degrade to
//     one link per step, never to a wrong answer.
//   * Up to 64 runs form a batch; the batch's values are decoded by the whole block (value i finds its run by binary search
//     in the batch's prefix sums).  part / nparts stripes the BATCHES of one page over several blocks: every block walks the
//     whole chain (cheap), but decodes only its own batches, so a page of a million values is not one block's job.
template <class Emit>
__device__ int64_t hybrid_decode(const uint8_t *__restrict__ p, int64_t nbytes, int bw, int64_t max_values, int part, int nparts, Emit emit) {
  __shared__ uint64_t s_arg[SCAN_RUNS];        // RLE: the value; packed: byte offset of the run's first group
  __shared__ uint8_t s_rle[SCAN_RUNS];
  __shared__ uint32_t s_pref[SCAN_RUNS + 1];
  __shared__ int s_nruns;
  __shared__ int64_t s_pos;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) s_pos = 0;
  __syncthreads();
  int64_t produced = 0;
  if (bw == 0) {   // a dictionary of one entry: every value is 0 (initFromPage :109-113)
    if (part == 0)
      for (int64_t i = tid; i < max_values; i += SCAN_THREADS) emit(i, 0ull);
    return max_values;
  }
  const int vbytes = (bw + 7) >> 3;
  for (int batch = 0; produced < max_values; batch++) {
    if (tid < 32) {
      int64_t pos = s_pos;
      int n = 0;
      int64_t acc = 0;
      const int64_t want = max_values - produced;
      if (lane == 0) s_pref[0] = 0;
      while (n < SCAN_RUNS && pos < nbytes && acc < want) {
        int hlen;
        const uint32_t header = read_uvarint(p, pos, nbytes, &hlen);
        const bool packed = header & 1;
        const int64_t c = packed ? (int64_t)(header >> 1) * 8 : (int64_t)(header >> 1);
        const int64_t run_bytes = hlen + (packed ? (int64_t)(header >> 1) * bw : vbytes);
        if (c <= 0) {   // empty run: nothing to decode, step over it
          pos += run_bytes;
          continue;
        }
        const int64_t q = pos + (int64_t)lane * run_bytes;
        bool same = lane == 0;
        if (lane > 0 && q + hlen <= nbytes) {
          int hl2;
          same = read_uvarint(p, q, nbytes, &hl2) == header && hl2 == hlen;
        }
        const uint32_t ball = __ballot_sync(0xffffffffu, same);
        int cnt = ball == 0xffffffffu ? 32 : __ffs(~ball) - 1;
        if (cnt > SCAN_RUNS - n) cnt = SCAN_RUNS - n;
        const int64_t needed = (want - acc + c - 1) / c;   // runs until the page's value count is reached
        if (cnt > needed) cnt = (int)needed;
        if (lane < cnt) {
          s_rle[n + lane] = packed ? 0 : 1;
          s_arg[n + lane] = packed ? (uint64_t)(q + hlen) : (q + hlen + vbytes <= nbytes ? load_le(p + q + hlen, vbytes) : 0);
          int64_t upto = acc + (int64_t)(lane + 1) * c;
          if (upto > want) upto = want;                    // the last packed group may be padded
          s_pref[n + lane + 1] = (uint32_t)upto;
        }
        n += cnt;
        pos += (int64_t)cnt * run_bytes;
        acc += (int64_t)cnt * c;
        if (acc > want) acc = want;
        if (acc >= (1ll << 30)) break;                     // keep the batch's prefix sums in 32 bits
      }
      if (lane == 0) {
        s_nruns = n;
        s_pos = pos;
      }
    }
    __syncthreads();
    const int nruns = s_nruns;
    const uint32_t total = nruns ? s_pref[nruns] : 0;
    if (nruns == 0 || total == 0) break;   // stream exhausted (malformed page: fewer values than announced)
    if (batch % nparts == part) {
      for (uint32_t i = tid; i < total; i += SCAN_THREADS) {
        int lo = 0, hi = nruns;               // last run with pref <= i
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (s_pref[mid] <= i) lo = mid; else hi = mid;
        }
        uint64_t v;
        if (s_rle[lo]) v = s_arg[lo];
        else {
          const uint64_t bit = (uint64_t)(i - s_pref[lo]) * (uint64_t)bw;
          const int64_t byte = (int64_t)s_arg[lo] + (int64_t)(bit >> 3);
          const int need = (int)(((bit & 7) + bw + 7) >> 3);
          const int avail = (int)(nbytes - byte < need ? (nbytes - byte > 0 ? nbytes - byte : 0) : need);
          v = (load_le(p + byte, avail) >> (bit & 7)) & ((bw >= 64) ? ~0ull : ((1ull << bw) - 1));
        }
        emit(produced + i, v);
      }
    }
    produced += total;
    __syncthreads();
  }
  return produced;
}

// definition levels of one page -> one validity byte per row (block-cooperative)
__device__ void decode_validity(const PageTask &pg, uint8_t *vb, bool page_nullable) {
  const int64_t n = pg.num_values;
  if (page_nullable) {
    const int64_t got = hybrid_decode(pg.def, pg.def_bytes, 1, n, 0, 1, [&](int64_t i, uint64_t v) { vb[i] = (uint8_t)(v & 1); });
    for (int64_t i = got + threadIdx.x; i < n; i += SCAN_THREADS) vb[i] = 0;
  } else {
    for (int64_t i = threadIdx.x; i < n; i += SCAN_THREADS) vb[i] = 1;
  }
  __syncthreads();
}

// value space -> row space: put(row, valid, idx) for every row of the page, idx = number of valid rows before it (a block
// scan of the validity bytes, PER rows per thread per tile)
template <class Put>
__device__ void expand_rows(const uint8_t *vb, int64_t n, Put put) {
  __shared__ int s_warp[SCAN_THREADS / 32];
  __shared__ int64_t s_base;
  const int tid = threadIdx.x;
  if (tid == 0) s_base = 0;
  __syncthreads();
  constexpr int PER = 4;
  for (int64_t tile = 0; tile < n; tile += SCAN_THREADS * PER) {
    const int64_t r0 = tile + (int64_t)tid * PER;
    int cnt = 0;
    uint8_t v[PER];
#pragma unroll
    for (int k = 0; k < PER; k++) {
      v[k] = r0 + k < n ? vb[r0 + k] : 0;
      cnt += v[k];
    }
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int o = __shfl_up_sync(0xffffffffu, incl, d);
      if ((tid & 31) >= d) incl += o;
    }
    if ((tid & 31) == 31) s_warp[tid >> 5] = incl;
    __syncthreads();
    int wbase = 0;
    for (int w = 0; w < (tid >> 5); w++) wbase += s_warp[w];
    int total = 0;
    for (int w = 0; w < SCAN_THREADS / 32; w++) total += s_warp[w];
    int64_t idx = s_base + wbase + incl - cnt;
#pragma unroll
    for (int k = 0; k < PER; k++) {
      if (r0 + k >= n) break;
      put(r0 + k, v[k] != 0, idx);
      if (v[k]) idx++;
    }
    __syncthreads();
    if (tid == 0) s_base += total;
    __syncthreads();
  }
}

// fixed-width values: row r of the page takes dense[#valid rows before r], NULL rows 0
__device__ void expand_fixed(const uint8_t *vb, int64_t n, const void *dense, void *dst_page, int ow) {
  expand_rows(vb, n, [&](int64_t r, bool valid, int64_t idx) {
    uint64_t val = 0;
    if (valid) {
      switch (ow) {
        case 1: val = ((const uint8_t *)dense)[idx]; break;
        case 2: val = ((const uint16_t *)dense)[idx]; break;
        case 4: val = ((const uint32_t *)dense)[idx]; break;
        default: val = ((const uint64_t *)dense)[idx]; break;
      }
    }
    store_value(dst_page, ow, r, val);
  });
}

// inclusive block scan of one 64-bit value per thread (wrapping); *total = sum over the block.  All threads call it.
__device__ __forceinline__ uint64_t block_scan_u64(uint64_t x, uint64_t *total) {
  __shared__ uint64_t s_w[SCAN_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t o = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += o;
  }
  if (lane == 31) s_w[tid >> 5] = x;
  __syncthreads();
  uint64_t base = 0, tot = 0;
  for (int w = 0; w < SCAN_THREADS / 32; w++) {
    if (w < (tid >> 5)) base += s_w[w];
    tot += s_w[w];
  }
  __syncthreads();
  *total = tot;
  return base + x;
}

// unsigned LEB128 of up to 64 bits (bounded by nbytes)
__device__ __forceinline__ uint64_t read_uvarint64(const uint8_t *__restrict__ p, int64_t pos, int64_t nbytes, int *len) {
  uint64_t v = 0;
  int shift = 0, l = 0;
  while (pos + l < nbytes) {
    const uint8_t b = p[pos + l++];
    if (shift < 64) v |= (uint64_t)(b & 0x7f) << shift;
    shift += 7;
    if (!(b & 0x80) || l >= 10) break;
  }
  *len = l;
  return v;
}
__device__ __forceinline__ uint64_t unzigzag(uint64_t u) { return (u >> 1) ^ (0ull - (u & 1)); }

// bw (<= 64) bits starting at bit `bit` of p[0..nbytes); bytes past the end read as 0
__device__ __forceinline__ uint64_t unpack_bits(const uint8_t *__restrict__ p, int64_t nbytes, uint64_t bit, int bw) {
  if (bw == 0) return 0;
  const int64_t byte = (int64_t)(bit >> 3);
  const int sh = (int)(bit & 7);
  const int need = (sh + bw + 7) >> 3;   // <= 9
  const int64_t left = nbytes - byte;
  const int lo_n = (int)(left <= 0 ? 0 : (left < 8 ? left : 8));
  uint64_t v = load_le(p + byte, lo_n < need ? lo_n : (need < 8 ? need : 8)) >> sh;
  if (need > 8 && left > 8) v |= (uint64_t)p[byte + 8] << (64 - sh);
  return bw >= 64 ? v : (v & ((1ull << bw) - 1));
}

// DELTA_BINARY_PACKED (VectorizedDeltaBinaryPackedReader.java): header <block size><miniblocks per block><total count><zig-zag first
// value>, then blocks of <zig-zag min delta><one bit-width byte per miniblock><packed miniblocks>; value i+1 = value i + min delta +
// packed delta, wrapping in 64 bits.  In the last block the bit-width bytes of unused miniblocks are present, their bodies are
// not.  Block-cooperative, in the manner of hybrid_decode: warp 0's lane 0 walks the miniblock headers (one byte each, plus a
// varint per block) into a batch of up to SCAN_RUNS miniblocks; the block decodes the batch's deltas (delta i finds its miniblock
// by binary search) and turns them into values with a block scan carried across tiles.  emit(i, v) for i < max_values (values the
// stream does not hold are emitted as 0); returns the byte position where the stream ends (the whole stream is walked, also when
// max_values is smaller), the same in every thread.
template <class Emit>
__device__ int64_t dbp_decode(const uint8_t *__restrict__ p, int64_t nbytes, int64_t max_values, Emit emit) {
  __shared__ int64_t s_off[SCAN_RUNS];      // byte offset of the miniblock's body
  __shared__ uint64_t s_min[SCAN_RUNS];
  __shared__ uint8_t s_bw[SCAN_RUNS];
  __shared__ uint32_t s_pref[SCAN_RUNS + 1];
  __shared__ int s_n;
  __shared__ int64_t s_pos, s_walked, s_bwpos, s_done_total, s_decoded;
  __shared__ uint64_t s_carry, s_bmin;
  __shared__ int s_m, s_minis, s_vpm;
  const int tid = threadIdx.x;
  if (tid == 0) {
    int l;
    int64_t pos = 0;
    const uint64_t block = read_uvarint64(p, pos, nbytes, &l); pos += l;
    const uint64_t minis = read_uvarint64(p, pos, nbytes, &l); pos += l;
    const uint64_t total = read_uvarint64(p, pos, nbytes, &l); pos += l;
    const uint64_t first = unzigzag(read_uvarint64(p, pos, nbytes, &l)); pos += l;
    // the page walker validated the header of every page it described; a hand-built descriptor gets the same limits here
    const bool ok = block >= 1 && block <= (1u << 20) && minis >= 1 && minis <= block && (block / minis) % 8 == 0 && block % minis == 0;
    s_minis = ok ? (int)minis : 1;
    s_vpm = ok ? (int)(block / minis) : 0;
    s_m = s_minis;                                   // no block open yet
    s_done_total = ok && total > 0 ? (int64_t)(total < (1ull << 40) ? total : (1ull << 40)) - 1 : 0;   // deltas in the stream
    s_walked = 0;
    s_pos = pos;
    s_carry = first;
    s_decoded = ok && total > 0 && max_values > 0 ? 1 : 0;
    if (s_decoded) emit(0, first);
  }
  __syncthreads();
  const int64_t want = max_values - 1;             // deltas to decode
  while (true) {
    if (tid == 0) {
      int n = 0;
      uint32_t acc = 0;
      int64_t pos = s_pos, walked = s_walked, bwpos = s_bwpos;
      int m = s_m;
      const int minis = s_minis, vpm = s_vpm;
      const int64_t total = s_done_total;
      uint64_t bmin = s_bmin;
      s_pref[0] = 0;
      while (walked < total && n < SCAN_RUNS && acc < (1u << 30)) {
        if (m == minis) {                            // next block: min delta, then the bit widths of all its miniblocks
          if (pos >= nbytes) { walked = total; break; }
          int l;
          bmin = unzigzag(read_uvarint64(p, pos, nbytes, &l));
          bwpos = pos + l;
          pos = bwpos + minis;
          m = 0;
        }
        int bw = bwpos + m < nbytes ? p[bwpos + m] : 0;
        if (bw > 64) bw = 64;
        const int64_t cnt = total - walked < vpm ? total - walked : vpm;
        if (walked < want) {
          const int64_t take = want - walked < cnt ? want - walked : cnt;
          s_off[n] = pos;
          s_min[n] = bmin;
          s_bw[n] = (uint8_t)bw;
          acc += (uint32_t)take;
          s_pref[n + 1] = acc;
          n++;
        }
        pos += (int64_t)vpm * bw / 8;                // a miniblock that holds any value is stored whole
        walked += cnt;
        m++;
      }
      s_n = n;
      s_pos = pos < nbytes ? pos : nbytes;
      s_walked = walked;
      s_bwpos = bwpos;
      s_m = m;
      s_bmin = bmin;
    }
    __syncthreads();
    const int nm = s_n;
    if (nm == 0) break;
    const uint32_t bt = s_pref[nm];
    const int64_t base = s_decoded;
    for (uint32_t t0 = 0; t0 < bt; t0 += SCAN_THREADS) {
      const uint32_t i = t0 + tid;
      uint64_t d = 0;
      if (i < bt) {
        int lo = 0, hi = nm;                         // last miniblock with pref <= i
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (s_pref[mid] <= i) lo = mid; else hi = mid;
        }
        const int bw = s_bw[lo];
        d = s_min[lo] + unpack_bits(p + s_off[lo], nbytes - s_off[lo], (uint64_t)(i - s_pref[lo]) * (uint64_t)bw, bw);
      }
      uint64_t tot;
      const uint64_t v = s_carry + block_scan_u64(d, &tot);
      if (i < bt) emit(base + i, v);
      __syncthreads();
      if (tid == 0) s_carry += tot;
      __syncthreads();
    }
    if (tid == 0) s_decoded += bt;
    __syncthreads();
  }
  for (int64_t i = s_decoded + tid; i < max_values; i += SCAN_THREADS) emit(i, 0ull);
  const int64_t end = s_pos;
  __syncthreads();
  return end;
}

// PLAIN byte arrays (VectorizedPlainValuesReader.readBinary): [4-byte LE length][bytes] per value.  The lengths form a chain, so
// one thread walks it, but over a window of the page staged in shared memory by the whole block: one HBM round trip per window,
// not per value.  A value larger than the window moves the next window to the length that follows it.  Lengths are clamped
// to the bytes left.  emit(k, offset of the bytes, length) for the first max_values values; returns how many there were.
constexpr int PLAIN_WINDOW = 8192;
template <class Emit>
__device__ int64_t plain_walk(const uint8_t *__restrict__ p, int64_t nbytes, int64_t max_values, Emit emit) {
  __shared__ uint8_t s_win[PLAIN_WINDOW];
  __shared__ int64_t s_pos, s_k;
  const int tid = threadIdx.x;
  if (tid == 0) {
    s_pos = 0;
    s_k = 0;
  }
  __syncthreads();
  while (true) {
    const int64_t w0 = s_pos, k0 = s_k;
    if (k0 >= max_values || w0 + 4 > nbytes) break;
    const int64_t wn = nbytes - w0 < PLAIN_WINDOW ? nbytes - w0 : PLAIN_WINDOW;
    for (int64_t i = tid; i < wn; i += SCAN_THREADS) s_win[i] = p[w0 + i];
    __syncthreads();
    if (tid == 0) {
      int64_t pos = w0, k = k0;
      while (k < max_values && pos + 4 <= nbytes && pos + 4 <= w0 + wn) {
        const uint8_t *h = s_win + (pos - w0);
        const int64_t len = (int64_t)((uint32_t)h[0] | ((uint32_t)h[1] << 8) | ((uint32_t)h[2] << 16) | ((uint32_t)h[3] << 24));
        const int64_t left = nbytes - pos - 4;
        const int64_t l = len < left ? len : left;
        emit(k, pos + 4, (int32_t)l);
        pos += 4 + l;
        k++;
      }
      s_pos = pos;
      s_k = k;
    }
    __syncthreads();
  }
  const int64_t got = s_k;
  __syncthreads();
  return got;
}

// number of non-zero validity bytes of a page
__device__ int64_t count_valid(const uint8_t *vb, int64_t n) {
  int64_t c = 0;
  for (int64_t i = threadIdx.x; i < n; i += SCAN_THREADS) c += vb[i];
  uint64_t tot;
  block_scan_u64((uint64_t)c, &tot);
  return (int64_t)tot;
}

// RLE_DICTIONARY values of a page: [bit width][hybrid runs of dictionary indices].  SCALED (TIMESTAMP(MILLIS)) is a template
// constant so that the other pages keep the hot loop they have without a multiplier.
template <bool SCALED>
__device__ __forceinline__ void dict_values(const PageTask &pg, const ColTask &c, void *dense, int part, int nparts) {
  const int bw = pg.values_bytes > 0 ? pg.values[0] : 0;
  const uint8_t *dict = c.dict;
  const int pw = c.phys_width, ow = c.out_width, dcount = c.dict_count, mul = SCALED ? c.mul : 0;
  hybrid_decode(pg.values + 1, pg.values_bytes - 1, bw, pg.num_values, part, nparts, [&](int64_t i, uint64_t idx) {
    uint64_t v = 0;
    if ((int64_t)idx < dcount) v = column_value(pw == 0 ? dict[idx] : load_le(dict + idx * pw, pw), pw, ow, mul);
    store_value(dense, ow, i, v);
  });
}

// (4 blocks per SM: the register budget the kernel had before the TIMESTAMP(MILLIS) path, at no spill)
__global__ void __launch_bounds__(SCAN_THREADS, 4) scan_decode_kernel(const PageTask *__restrict__ pages, const ColTask *__restrict__ cols, int nparts) {
  const PageTask pg = pages[blockIdx.x / nparts];
  int part = blockIdx.x % nparts;
  const ColTask c = cols[pg.col];
  const int64_t n = pg.num_values;
  // ---- (1) definition levels -> validity bytes -------------------------------------------------------------------------
  uint8_t *vb = c.valid_bytes ? c.valid_bytes + pg.row_start : nullptr;
  const bool page_nullable = pg.def != nullptr && pg.def_bytes > 0;
  if (page_nullable || pg.encoding != SB_ENC_RLE_DICTIONARY) {   // only hybrid-encoded, NULL-free pages are striped over several blocks
    if (part != 0) return;
    nparts = 1;
  }
  if (vb && part == 0) decode_validity(pg, vb, page_nullable);
  const int tid = threadIdx.x;
  // ---- (2) values -> dense value space (or straight to the output when the page has no NULLs) -----------------------------
  void *dst_page = (uint8_t *)c.out + pg.row_start * c.out_width;
  void *dense = page_nullable ? (void *)(c.dense + pg.row_start * c.out_width) : dst_page;
  const int ow = c.out_width;
  if (pg.encoding == SB_ENC_PLAIN) {
    if (c.phys_width == 0) {   // BOOLEAN: bit-packed, LSB first
      const int64_t avail = pg.values_bytes * 8 < n ? pg.values_bytes * 8 : n;
      for (int64_t i = tid; i < avail; i += SCAN_THREADS) ((uint8_t *)dense)[i] = (pg.values[i >> 3] >> (i & 7)) & 1;
    } else {
      const int pw = c.phys_width;
      const int64_t avail = pg.values_bytes / pw < n ? pg.values_bytes / pw : n;
      if (pw == ow && c.mul <= 1 && ((((uintptr_t)pg.values) | ((uintptr_t)dense)) & 15) == 0) {   // straight copy, 16 bytes per thread
        const int64_t bytes = avail * pw, vec = bytes >> 4;
        const uint4 *s4 = (const uint4 *)pg.values;
        uint4 *d4 = (uint4 *)dense;
        for (int64_t i = tid; i < vec; i += SCAN_THREADS) d4[i] = s4[i];
        for (int64_t i = (vec << 4) + tid; i < bytes; i += SCAN_THREADS) ((uint8_t *)dense)[i] = pg.values[i];
      } else {
        for (int64_t i = tid; i < avail; i += SCAN_THREADS) {
          store_value(dense, ow, i, column_value(load_le(pg.values + i * pw, pw), pw, ow, c.mul));
        }
      }
    }
  } else if (pg.encoding == SB_ENC_RLE_BOOLEAN) {   // BOOLEAN values as RLE (data page V2 writers): [4-byte length][hybrid, bit width 1]
    if (pg.values_bytes > 4)
      hybrid_decode(pg.values + 4, pg.values_bytes - 4, 1, n, 0, 1, [&](int64_t i, uint64_t v) { ((uint8_t *)dense)[i] = (uint8_t)(v & 1); });
  } else if (c.mul > 1) {   // RLE_DICTIONARY: [bit width][hybrid runs of dictionary indices]
    dict_values<true>(pg, c, dense, part, nparts);
  } else {
    dict_values<false>(pg, c, dense, part, nparts);
  }
  if (!page_nullable) return;
  __syncthreads();
  // ---- (3) expand value space -> row space: row r takes dense[#valid rows before r] --------------------------------------
  expand_fixed(vb, n, dense, dst_page, ow);
}

// DELTA_BINARY_PACKED pages of INT32 / INT64 columns, one block per page, steps (1)-(3) of scan_decode_kernel around dbp_decode
// (a kernel of its own so that the hybrid decoder's kernel keeps its registers)
__global__ void __launch_bounds__(SCAN_THREADS) scan_delta_kernel(const PageTask *__restrict__ pages, const ColTask *__restrict__ cols) {
  const PageTask pg = pages[blockIdx.x];
  const ColTask c = cols[pg.col];
  const int64_t n = pg.num_values;
  uint8_t *vb = c.valid_bytes ? c.valid_bytes + pg.row_start : nullptr;
  const bool page_nullable = pg.def != nullptr && pg.def_bytes > 0;
  if (vb) decode_validity(pg, vb, page_nullable);
  const int ow = c.out_width, pw = c.phys_width, mul = c.mul;
  void *dst_page = (uint8_t *)c.out + pg.row_start * ow;
  void *dense = page_nullable ? (void *)(c.dense + pg.row_start * ow) : dst_page;
  dbp_decode(pg.values, pg.values_bytes, n, [&](int64_t i, uint64_t v) {   // 64-bit running sum, truncated to the column's width
    store_value(dense, ow, i, column_value(v, pw, ow, mul));
  });
  if (!page_nullable) return;
  __syncthreads();
  expand_fixed(vb, n, dense, dst_page, ow);
}

// ---- BYTE_ARRAY -> SB_STRING --------------------------------------------------------------------------------------------
// (a) str_dict_kernel: one block per dictionary chunk walks its PLAIN dictionary page into (offset, length) entries.
// (b) str_page_kernel: one block per page: validity, then every value's (length, source offset in the chunk, prefix length) in
//     value space, expanded to row space (NULL rows: length 0).
// (c) host: exclusive scan of the lengths -> int64 offsets; ONE stream synchronisation reads back the arena sizes of all string
//     columns of the call (Column::string_bytes is exact on the host); an arena above 2^31 - 1 bytes is refused.
// (d) str_copy_kernel: row-parallel, one warp per 32 rows: the bytes each value takes from its page (DELTA_BYTE_ARRAY: the
//     suffix, after the prefix) and the int32 offsets.
// (e) str_prefix_kernel: one warp per DELTA_BYTE_ARRAY page, in value order: value i's first prefix[i] bytes from value i-1.
struct StrColTask {
  const uint8_t *base;                 // device chunk
  uint8_t *valid_bytes;                // or nullptr
  int32_t *vlen, *vpre;                // value space (NULLable columns) or the row arrays themselves
  int64_t *vsrc;
  int32_t *rlen, *rpre;                // row space; rpre nullptr unless a page is DELTA_BYTE_ARRAY
  int64_t *rsrc;
  int32_t *dict_len;                   // dictionary entries
  int64_t *dict_src;
  int64_t dict_offset, data_bytes;
  int32_t dict_count;
  int32_t pad;
};
struct StrOutTask {
  const int64_t *off;                  // exclusive scan of rlen
  int32_t *out_off;                    // column offsets (rows + 1)
  uint8_t *arena;
  int64_t nrows;
};

__global__ void __launch_bounds__(SCAN_THREADS) str_dict_kernel(const StrColTask *__restrict__ cols, const int32_t *__restrict__ which) {
  const StrColTask c = cols[which[blockIdx.x]];
  const int64_t got = plain_walk(c.base + c.dict_offset, c.data_bytes - c.dict_offset, c.dict_count, [&](int64_t k, int64_t off, int32_t len) {
    c.dict_len[k] = len;
    c.dict_src[k] = c.dict_offset + off;
  });
  for (int64_t k = got + threadIdx.x; k < c.dict_count; k += SCAN_THREADS) {
    c.dict_len[k] = 0;
    c.dict_src[k] = 0;
  }
}

// DELTA_LENGTH_BYTE_ARRAY section at p[0..nbytes): lengths, then the bytes; lens[i] clamped so that value i lies inside the section.
// Writes lens / src (chunk offsets: p is at chunk offset p_off) for i < nvals; returns the section's end.
__device__ int64_t dlba_decode(const uint8_t *p, int64_t nbytes, int64_t p_off, int64_t nvals, int32_t *lens, int64_t *src) {
  const int64_t start = dbp_decode(p, nbytes, nvals, [&](int64_t i, uint64_t v) {
    lens[i] = (int64_t)v < 0 ? 0 : ((int64_t)v > 0x7fffffff ? 0x7fffffff : (int32_t)v);
  });
  __syncthreads();
  __shared__ int64_t s_run;
  if (threadIdx.x == 0) s_run = start;
  __syncthreads();
  for (int64_t t0 = 0; t0 < nvals; t0 += SCAN_THREADS) {
    const int64_t i = t0 + threadIdx.x;
    const int64_t l = i < nvals ? lens[i] : 0;
    uint64_t tot;
    const int64_t at = s_run + (int64_t)block_scan_u64((uint64_t)l, &tot) - l;
    if (i < nvals) {
      const int64_t s = at < nbytes ? at : nbytes;
      lens[i] = (int32_t)(s + l <= nbytes ? l : nbytes - s);
      src[i] = p_off + s;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_run += (int64_t)tot;
    __syncthreads();
  }
  const int64_t end = s_run < nbytes ? s_run : nbytes;
  __syncthreads();
  return end;
}

__global__ void __launch_bounds__(SCAN_THREADS) str_page_kernel(const PageTask *__restrict__ pages, const StrColTask *__restrict__ cols) {
  const PageTask pg = pages[blockIdx.x];
  const StrColTask c = cols[pg.col];
  const int64_t n = pg.num_values;
  uint8_t *vb = c.valid_bytes ? c.valid_bytes + pg.row_start : nullptr;
  const bool page_nullable = pg.def != nullptr && pg.def_bytes > 0;
  if (vb) decode_validity(pg, vb, page_nullable);
  const int64_t nvals = page_nullable ? count_valid(vb, n) : n;
  int32_t *vlen = (page_nullable ? c.vlen : c.rlen) + pg.row_start;
  int64_t *vsrc = (page_nullable ? c.vsrc : c.rsrc) + pg.row_start;
  int32_t *vpre = c.rpre ? (page_nullable ? c.vpre : c.rpre) + pg.row_start : nullptr;
  const int64_t voff = pg.values - c.base;   // chunk offset of the page's values
  int64_t got = nvals;
  if (pg.encoding == SB_ENC_PLAIN) {
    got = plain_walk(pg.values, pg.values_bytes, nvals, [&](int64_t k, int64_t off, int32_t len) {
      vlen[k] = len;
      vsrc[k] = voff + off;
    });
  } else if (pg.encoding == SB_ENC_RLE_DICTIONARY) {
    const int bw = pg.values_bytes > 0 ? pg.values[0] : 0;
    got = nvals > 0 ? hybrid_decode(pg.values + 1, pg.values_bytes - 1, bw > 32 ? 32 : bw, nvals, 0, 1, [&](int64_t i, uint64_t idx) {
      const bool in = idx < (uint64_t)c.dict_count;
      vlen[i] = in ? c.dict_len[idx] : 0;
      vsrc[i] = in ? c.dict_src[idx] : 0;
    }) : 0;
  } else if (pg.encoding == SB_ENC_DELTA_LENGTH_BYTE_ARRAY) {
    dlba_decode(pg.values, pg.values_bytes, voff, nvals, vlen, vsrc);
  } else {   // DELTA_BYTE_ARRAY: prefix lengths, then DELTA_LENGTH_BYTE_ARRAY suffixes; the length is prefix + suffix
    const int64_t pend = dbp_decode(pg.values, pg.values_bytes, nvals, [&](int64_t i, uint64_t v) {
      vpre[i] = (int64_t)v < 0 ? 0 : ((int64_t)v > 0x7fffffff ? 0x7fffffff : (int32_t)v);
    });
    dlba_decode(pg.values + pend, pg.values_bytes - pend, voff + pend, nvals, vlen, vsrc);
    for (int64_t i = threadIdx.x; i < nvals; i += SCAN_THREADS) {
      const int64_t l = (int64_t)vlen[i] + vpre[i];
      vlen[i] = (int32_t)(l > 0x7fffffff ? 0x7fffffff : l);
    }
  }
  for (int64_t i = got + threadIdx.x; i < nvals; i += SCAN_THREADS) {   // values the page does not hold are empty
    vlen[i] = 0;
    vsrc[i] = 0;
  }
  if (vpre && pg.encoding != SB_ENC_DELTA_BYTE_ARRAY)
    for (int64_t i = threadIdx.x; i < nvals; i += SCAN_THREADS) vpre[i] = 0;
  if (!page_nullable) return;
  __syncthreads();
  int32_t *rlen = c.rlen + pg.row_start, *rpre = c.rpre ? c.rpre + pg.row_start : nullptr;
  int64_t *rsrc = c.rsrc + pg.row_start;
  expand_rows(vb, n, [&](int64_t r, bool valid, int64_t idx) {
    rlen[r] = valid ? vlen[idx] : 0;
    rsrc[r] = valid ? vsrc[idx] : 0;
    if (rpre) rpre[r] = valid ? vpre[idx] : 0;
  });
}

// bytes that come from the page: value r's [pre, len) from its source; 8 loads in flight per lane
__global__ void __launch_bounds__(SCAN_THREADS) str_copy_kernel(StrColTask c, StrOutTask o) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * SCAN_THREADS + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * SCAN_THREADS) >> 5;
  for (int64_t r0 = warp * 32; r0 < o.nrows; r0 += nwarps * 32) {
    const int64_t r = r0 + lane;
    int64_t off = 0, src = 0;
    int32_t len = 0, pre = 0;
    if (r < o.nrows) {
      off = o.off[r];
      len = c.rlen[r];
      src = c.rsrc[r];
      pre = c.rpre ? c.rpre[r] : 0;
      if (pre > len) pre = len;
      o.out_off[r] = (int32_t)off;
    }
    const int rows = o.nrows - r0 < 32 ? (int)(o.nrows - r0) : 32;
    for (int k = 0; k < rows; k++) {
      const int64_t koff = __shfl_sync(0xffffffffu, off, k) + __shfl_sync(0xffffffffu, pre, k);
      const int64_t ksrc = __shfl_sync(0xffffffffu, src, k);
      const int64_t klen = __shfl_sync(0xffffffffu, len, k) - __shfl_sync(0xffffffffu, pre, k);
      const uint8_t *s = c.base + ksrc;
      uint8_t *d = o.arena + koff;
      for (int64_t b = lane; b < klen; b += 32 * 8) {
        uint8_t v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = b + 32 * u < klen ? s[b + 32 * u] : 0;
#pragma unroll
        for (int u = 0; u < 8; u++)
          if (b + 32 * u < klen) d[b + 32 * u] = v[u];
      }
    }
  }
}

// DELTA_BYTE_ARRAY prefixes, one warp per page in value order (VectorizedDeltaByteArrayReader.readValues): value i's first
// prefix[i] bytes are value i-1's.  A prefix longer than the previous value (a malformed page) is filled with zero bytes.
__global__ void str_prefix_kernel(const PageTask *__restrict__ pages, const StrColTask *__restrict__ cols, const StrOutTask *__restrict__ outs) {
  const PageTask pg = pages[blockIdx.x];
  const StrColTask c = cols[pg.col];
  const StrOutTask o = outs[pg.col];
  const int lane = threadIdx.x & 31;
  int64_t prev_off = 0, prev_len = 0;
  bool have_prev = false;
  for (int64_t r0 = pg.row_start; r0 < pg.row_start + pg.num_values; r0 += 32) {
    const int64_t r = r0 + lane;
    const bool in = r < pg.row_start + pg.num_values;
    const bool valid = in && (!c.valid_bytes || c.valid_bytes[r]);
    const int64_t off = in ? o.off[r] : 0;
    const int32_t len = in ? c.rlen[r] : 0, pre = in ? c.rpre[r] : 0;
    const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
    for (int k = 0; k < 32; k++) {
      if (!((vmask >> k) & 1)) continue;
      const int64_t koff = __shfl_sync(0xffffffffu, off, k);
      const int32_t klen = __shfl_sync(0xffffffffu, len, k);
      int32_t kpre = __shfl_sync(0xffffffffu, pre, k);
      if (kpre > klen) kpre = klen;
      for (int32_t b = lane; b < kpre; b += 32) o.arena[koff + b] = have_prev && b < prev_len ? o.arena[prev_off + b] : 0;
      __syncwarp();
      prev_off = koff;
      prev_len = klen;
      have_prev = true;
    }
  }
}

// ---- write side (tests, bench.py): dictionary indices of a sorted dictionary + bit packing into hybrid runs --------------
// One block per page of page_rows rows.  A page is [bit width byte] + bit-packed runs of 504 values (header 0x7F, the run
// length parquet-mr's RunLengthBitPackingHybridEncoder emits: 63 groups of 8) + one shorter last run, padded to 8 values.
template <typename T>
__global__ void __launch_bounds__(SCAN_THREADS) encode_dict_pages_kernel(const T *__restrict__ col, int64_t n, const T *__restrict__ dict, int32_t dcount,
                                                                         int bw, int64_t page_rows, int64_t page_stride, uint8_t *__restrict__ out) {
  const int64_t page = blockIdx.x;
  const int64_t r_lo = page * page_rows, r_hi = r_lo + page_rows < n ? r_lo + page_rows : n;
  uint8_t *dst = out + page * page_stride;
  if (threadIdx.x == 0) dst[0] = (uint8_t)bw;
  const int64_t rows = r_hi - r_lo;
  const int64_t full_runs = rows / 504, tail = rows - full_runs * 504;
  const int64_t run_bytes = 1 + 63 * (int64_t)bw;
  // one thread per group of 8 values: writes bw bytes
  const int64_t groups = (rows + 7) / 8;
  for (int64_t g = threadIdx.x; g < groups; g += SCAN_THREADS) {
    const int64_t run = g / 63, gin = g - run * 63;
    uint8_t *rp = dst + 1 + run * run_bytes;
    if (gin == 0) {
      const int64_t groups_in_run = run < full_runs ? 63 : (tail + 7) / 8;
      rp[0] = (uint8_t)((groups_in_run << 1) | 1);
    }
    uint8_t *gp = rp + 1 + gin * bw;
    uint64_t acc = 0;
    int nbits = 0, ob = 0;
    for (int k = 0; k < 8; k++) {
      const int64_t r = r_lo + g * 8 + k;
      uint64_t idx = 0;
      if (r < r_hi) {
        const T v = col[r];
        int lo = 0, hi = dcount;   // first dict entry >= v (dict is sorted, v is present)
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (dict[mid] < v) lo = mid + 1; else hi = mid;
        }
        idx = (uint64_t)lo;
      }
      acc |= idx << nbits;           // nbits < 8 here and bw <= 24: fits 64 bits
      nbits += bw;
      while (nbits >= 8) {
        gp[ob++] = (uint8_t)acc;
        acc >>= 8;
        nbits -= 8;
      }
    }
  }
}

}  // namespace sb

using namespace sb;

// ---- host: Thrift compact protocol reader for Parquet PageHeader (parquet-format/src/main/thrift/parquet.thrift) ------------
namespace {
struct Thrift {
  const uint8_t *p, *end;
  bool ok = true;
  uint64_t varint() {
    uint64_t v = 0;
    int shift = 0;
    while (p < end) {
      const uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
      shift += 7;
      if (shift > 63) break;
    }
    ok = false;
    return 0;
  }
  int64_t zigzag() {
    const uint64_t u = varint();
    return (int64_t)(u >> 1) ^ -(int64_t)(u & 1);
  }
  void skip(int type);
  void skip_struct() {
    int16_t last = 0;
    while (ok && p < end) {
      const uint8_t b = *p++;
      if (b == 0) return;
      const int type = b & 0x0f, delta = b >> 4;
      if (delta) last = (int16_t)(last + delta); else last = (int16_t)zigzag();
      skip(type);
    }
    ok = false;
  }
};
void Thrift::skip(int type) {
  switch (type) {
    case 1: case 2: break;                                  // BOOLEAN_TRUE / FALSE (value in the type nibble)
    case 3: p += 1; break;                                  // BYTE
    case 4: case 5: case 6: varint(); break;                // I16 / I32 / I64 (zigzag varints)
    case 7: p += 8; break;                                  // DOUBLE
    case 8: { const uint64_t n = varint(); p += n; break; } // BINARY
    case 9: case 10: {                                      // LIST / SET
      if (p >= end) { ok = false; return; }
      const uint8_t h = *p++;
      uint64_t n = h >> 4;
      const int et = h & 0x0f;
      if (n == 15) n = varint();
      for (uint64_t i = 0; i < n && ok; i++) {
        if (et == 1 || et == 2) p += 1; else skip(et);      // booleans inside lists take one byte each
      }
      break;
    }
    case 11: {                                              // MAP
      const uint64_t n = varint();
      if (n) {
        if (p >= end) { ok = false; return; }
        const uint8_t kv = *p++;
        for (uint64_t i = 0; i < n && ok; i++) { skip(kv >> 4); skip(kv & 0x0f); }
      }
      break;
    }
    case 12: skip_struct(); break;
    default: ok = false;
  }
  if (p > end) ok = false;
}

struct PageHeader {
  int32_t type = -1, uncompressed = 0, compressed = 0;
  int32_t num_values = 0, encoding = -1, def_enc = -1, rep_enc = -1;     // data page v1 / v2 / dictionary
  int32_t num_nulls = 0, num_rows = 0, def_len = 0, rep_len = 0;
  bool v2_compressed = true, is_v2 = false;
};
// reads the fields of one nested header struct we care about
void read_inner(Thrift &t, PageHeader &h, int which) {   // which: 5 data v1, 7 dictionary, 8 data v2
  int16_t last = 0;
  while (t.ok && t.p < t.end) {
    const uint8_t b = *t.p++;
    if (b == 0) return;
    const int type = b & 0x0f, delta = b >> 4;
    if (delta) last = (int16_t)(last + delta); else last = (int16_t)t.zigzag();
    if (type == 5 || type == 4 || type == 6) {
      const int32_t v = (int32_t)t.zigzag();
      if (which == 5) { if (last == 1) h.num_values = v; else if (last == 2) h.encoding = v; else if (last == 3) h.def_enc = v; else if (last == 4) h.rep_enc = v; }
      else if (which == 7) { if (last == 1) h.num_values = v; else if (last == 2) h.encoding = v; }
      else { if (last == 1) h.num_values = v; else if (last == 2) h.num_nulls = v; else if (last == 3) h.num_rows = v; else if (last == 4) h.encoding = v;
             else if (last == 5) h.def_len = v; else if (last == 6) h.rep_len = v; }
    } else if ((type == 1 || type == 2) && which == 8 && last == 7) {
      h.v2_compressed = type == 1;
    } else t.skip(type);
  }
  t.ok = false;
}
bool read_page_header(Thrift &t, PageHeader &h) {
  int16_t last = 0;
  while (t.ok && t.p < t.end) {
    const uint8_t b = *t.p++;
    if (b == 0) return t.ok;
    const int type = b & 0x0f, delta = b >> 4;
    if (delta) last = (int16_t)(last + delta); else last = (int16_t)t.zigzag();
    if (type == 5 && last <= 3) {
      const int32_t v = (int32_t)t.zigzag();
      if (last == 1) h.type = v; else if (last == 2) h.uncompressed = v; else h.compressed = v;
    } else if (type == 12 && (last == 5 || last == 7 || last == 8)) {
      if (last == 8) h.is_v2 = true;
      read_inner(t, h, last);
    } else t.skip(type);
  }
  return false;
}

// The DELTA_BINARY_PACKED header in front of a DELTA_* page's values, validated as VectorizedDeltaBinaryPackedReader.initFromPage
// does (:91-122); for DELTA_BYTE_ARRAY it is the prefix-length stream's.  That stream's first value is the first prefix length:
// a page that does not start it at 0 continues the previous page's last value (PARQUET-246, VectorizedDeltaByteArrayReader
// :76-80), which the per-page decode does not carry over, so the page is refused instead.
void check_delta_header(const uint8_t *p, int64_t nbytes, int32_t enc, int64_t page_values, int page, int64_t page_pos) {
  Thrift t{p, p + nbytes};
  const uint64_t block = t.varint(), minis = t.varint(), total = t.varint();
  const int64_t first = t.zigzag();
  if (!t.ok) fail(SB_ERR_INVALID, "page %d (byte %lld of the column chunk): truncated DELTA_BINARY_PACKED header", page, (long long)page_pos);
  if (block < 1 || block > (1u << 20))
    fail(SB_ERR_INVALID, "page %d (byte %lld of the column chunk): DELTA_BINARY_PACKED block size %llu is not in [1, 2^20]", page, (long long)page_pos,
         (unsigned long long)block);
  if (minis < 1 || minis > block)
    fail(SB_ERR_INVALID, "page %d (byte %lld of the column chunk): DELTA_BINARY_PACKED miniblock count %llu is not in [1, %llu]", page,
         (long long)page_pos, (unsigned long long)minis, (unsigned long long)block);
  if (block % minis != 0 || (block / minis) % 8 != 0)
    fail(SB_ERR_INVALID, "page %d (byte %lld of the column chunk): DELTA_BINARY_PACKED miniblock size %llu / %llu is not a multiple of 8", page,
         (long long)page_pos, (unsigned long long)block, (unsigned long long)minis);
  if (total > (uint64_t)page_values)
    fail(SB_ERR_INVALID, "page %d (byte %lld of the column chunk): DELTA_BINARY_PACKED total count %llu exceeds the page's %lld values", page,
         (long long)page_pos, (unsigned long long)total, (long long)page_values);
  if (enc == SB_ENC_DELTA_BYTE_ARRAY && total > 0 && first != 0)
    fail(SB_ERR_UNSUPPORTED, "page %d (byte %lld of the column chunk): DELTA_BYTE_ARRAY page starts with prefix length %lld; continuing the "
         "previous page's value (PARQUET-246) is not supported", page, (long long)page_pos, (long long)first);
}

// SB_ENC_* of a data page's Parquet encoding
int32_t page_encoding(int32_t parquet_encoding) {
  switch (parquet_encoding) {
    case 0: return SB_ENC_PLAIN;
    case 2: case 8: return SB_ENC_RLE_DICTIONARY;
    case 3: return SB_ENC_RLE_BOOLEAN;   // only BOOLEAN columns may use it (checked in sb_scan_decode)
    case 5: return SB_ENC_DELTA_BINARY_PACKED;
    case 6: return SB_ENC_DELTA_LENGTH_BYTE_ARRAY;
    case 7: return SB_ENC_DELTA_BYTE_ARRAY;
  }
  fail(SB_ERR_UNSUPPORTED, "Parquet value encoding %d is not supported (PLAIN, RLE_DICTIONARY and the DELTA encodings are)", parquet_encoding);
}

// the checks a data page's header alone decides
void check_data_page_header(const PageHeader &h, int32_t max_def_level) {
  if (h.type == 0) {
    if (max_def_level > 0) SB_REQUIRE(h.def_enc == 3, "definition levels must be RLE encoded (got %d)", h.def_enc);
  } else {
    SB_REQUIRE(h.rep_len == 0, "repeated fields are not supported");
  }
}

// Levels and values of one data page whose body (as decoded) is [body, body + body_bytes) of the chunk: a V1 page of an optional
// column starts with the 4-byte length of its definition levels (`len4`; nullptr when the body is shorter), a V2 page gives the
// length in its header.
void data_page_sections(sb_page &pg, bool v1, int32_t max_def_level, int32_t v2_def_len, int64_t body, int64_t body_bytes, const uint8_t *len4) {
  int64_t vpos = body;
  const int64_t vend = body + body_bytes;
  if (v1) {
    if (max_def_level > 0) {   // [4-byte length][RLE definition levels]
      SB_REQUIRE(len4 != nullptr, "truncated definition levels");
      const uint32_t len = (uint32_t)len4[0] | ((uint32_t)len4[1] << 8) | ((uint32_t)len4[2] << 16) | ((uint32_t)len4[3] << 24);
      pg.def_offset = vpos + 4;
      pg.def_bytes = len;
      vpos += 4 + (int64_t)len;
    }
  } else {
    if (v2_def_len > 0) {
      pg.def_offset = vpos;
      pg.def_bytes = v2_def_len;
    }
    vpos += v2_def_len;
  }
  SB_REQUIRE(vpos <= vend, "Parquet page levels overrun the page");
  pg.values_offset = vpos;
  pg.values_bytes = vend - vpos;
}

// The page header walk of a chunk as it lies in a file ([dictionary_page_offset or data_page_offset, + total_compressed_size) of
// the column's metadata): calls page(span) for each dictionary and data page that passes the checks of every path, in order, and
// skips INDEX_PAGE and unknown types.  `cap` bounds the pages passed on (data pages only unless cap_dictionary).
// refuse_compressed: a page whose two sizes differ is SB_ERR_UNSUPPORTED unless it is a V2 page marked uncompressed.
template <class Page>
void walk_pages(const uint8_t *chunk, int64_t nbytes, int32_t codec, int32_t max_def_level, bool refuse_compressed, int32_t cap,
                bool cap_dictionary, Page page) {
  SB_REQUIRE(max_def_level == 0 || max_def_level == 1, "nested schemas are not supported (max definition level %d)", max_def_level);
  int32_t counted = 0;
  for (int64_t pos = 0, next; pos < nbytes; pos = next) {
    Thrift t{chunk + pos, chunk + nbytes};
    PageHeader h;
    if (!read_page_header(t, h)) fail(SB_ERR_INVALID, "malformed Parquet page header at byte %lld of the column chunk", (long long)pos);
    const int64_t body = t.p - chunk;
    const bool stored = h.is_v2 && !h.v2_compressed;
    if (refuse_compressed && h.compressed != h.uncompressed && !stored)
      fail(SB_ERR_UNSUPPORTED, "compressed Parquet pages are not decoded on this path (page at byte %lld: %d -> %d bytes)", (long long)pos,
           h.compressed, h.uncompressed);
    SB_REQUIRE(h.compressed >= 0 && h.uncompressed >= 0 && body + h.compressed <= nbytes, "Parquet page at byte %lld overruns the column chunk",
               (long long)pos);
    next = body + h.compressed;
    if (h.type != 0 && h.type != 2 && h.type != 3) continue;
    if (h.type != 2 || cap_dictionary) {
      SB_REQUIRE(counted < cap, "more than %d pages in the column chunk", cap);
      counted++;
    }
    SB_REQUIRE(h.num_values >= 0, "Parquet page at byte %lld has a negative value count (%d)", (long long)pos, h.num_values);
    sb_page_span sp;
    memset(&sp, 0, sizeof(sp));
    sp.page_type = h.type;
    sp.num_values = h.num_values;
    sp.body_offset = body;
    sp.header_bytes = (int32_t)(body - pos);
    sp.compressed_bytes = h.compressed;
    sp.uncompressed_bytes = h.uncompressed;
    sp.values_compressed = codec != SB_CODEC_UNCOMPRESSED && !stored;
    if (h.type == 2) {
      SB_REQUIRE(h.encoding == 0 || h.encoding == 2, "dictionary page encoding %d is not PLAIN", h.encoding);
      sp.encoding = SB_ENC_PLAIN;
    } else {
      sp.encoding = page_encoding(h.encoding);
      check_data_page_header(h, max_def_level);
      if (h.type == 3) sp.levels_bytes = h.def_len;
    }
    SB_REQUIRE(sp.levels_bytes >= 0 && sp.levels_bytes <= h.uncompressed && sp.levels_bytes <= h.compressed, "Parquet page levels overrun the page");
    if (!sp.values_compressed)
      SB_REQUIRE(h.compressed == h.uncompressed, "uncompressed Parquet page at byte %lld: %d stored bytes for %d", (long long)pos, h.compressed,
                 h.uncompressed);
    page(sp);
  }
}

// The sb_page descriptors and dictionary of one chunk, added span by span in page order (the last dictionary page counts), on
// both paths, so a page is refused with the same message whether or not it was compressed.  body: where the decoded body starts
// among the bytes the descriptors index; len4: its first 4 bytes (a V1 page's level length), nullptr when it is shorter;
// values_head(pg): the first bytes of pg's values, where a DELTA_* header starts, and how many of them can be read.
struct ChunkPages {
  std::vector<sb_page> pages;
  int64_t dict_offset = -1;
  int32_t dict_count = 0;

  template <class Head>
  void add(const sb_page_span &sp, int32_t max_def_level, int64_t body, const uint8_t *len4, Head values_head) {
    if (sp.page_type == 2) {
      dict_offset = body;
      dict_count = sp.num_values;
      return;
    }
    sb_page pg;
    memset(&pg, 0, sizeof(pg));
    pg.encoding = sp.encoding;
    pg.num_values = sp.num_values;
    data_page_sections(pg, sp.page_type == 0, max_def_level, sp.levels_bytes, body, sp.uncompressed_bytes, len4);
    if (pg.encoding >= SB_ENC_DELTA_BINARY_PACKED) {
      const std::pair<const uint8_t *, int64_t> head = values_head(pg);
      check_delta_header(head.first, head.second, pg.encoding, pg.num_values, (int)pages.size(), sp.body_offset - sp.header_bytes);
    }
    pages.push_back(pg);
  }
};
}  // namespace

static void require_codec(int32_t codec) {
  static const char *const names[] = {"UNCOMPRESSED", "SNAPPY", "GZIP", "LZO", "BROTLI", "LZ4", "ZSTD", "LZ4_RAW"};
  if (codec == SB_CODEC_UNCOMPRESSED || codec == SB_CODEC_SNAPPY) return;
  if (codec > 0 && codec < 8) fail(SB_ERR_UNSUPPORTED, "Parquet compression codec %s is not supported by the GPU scan (UNCOMPRESSED and SNAPPY are)", names[codec]);
  fail(SB_ERR_UNSUPPORTED, "Parquet compression codec %d is not supported by the GPU scan (UNCOMPRESSED and SNAPPY are)", codec);
}

// Host only (no device needed): the descriptors sb_scan_decode takes for one column chunk as it lies in a Parquet file.
// max_def_level: 0 for a required column, 1 for an optional one.
extern "C" int sb_parquet_chunk_pages(const uint8_t *chunk, int64_t nbytes, int32_t max_def_level, sb_page *out_pages, int32_t pages_cap,
                                      int32_t *out_npages, int64_t *out_dict_offset, int32_t *out_dict_count) {
  SB_API_BEGIN
  SB_REQUIRE(chunk && out_pages && out_npages && out_dict_offset && out_dict_count && nbytes >= 0, "null argument");
  ChunkPages cp;
  walk_pages(chunk, nbytes, SB_CODEC_UNCOMPRESSED, max_def_level, true, pages_cap, false, [&](const sb_page_span &sp) {
    cp.add(sp, max_def_level, sp.body_offset, sp.uncompressed_bytes >= 4 ? chunk + sp.body_offset : nullptr,
           [&](const sb_page &pg) { return std::make_pair(chunk + pg.values_offset, pg.values_bytes); });
  });
  std::copy(cp.pages.begin(), cp.pages.end(), out_pages);
  *out_npages = (int32_t)cp.pages.size();
  *out_dict_offset = cp.dict_offset;
  *out_dict_count = cp.dict_count;
  SB_API_END
}

// Host only: the spans of a chunk whose pages may be compressed.  Unlike sb_parquet_chunk_pages it never looks inside a body:
// whether a page is compressed comes from the footer's codec (a Snappy page may compress to exactly its own size, and tiny
// pages grow), and the levels and DELTA headers are checked once the device has decoded the bodies.
extern "C" int sb_parquet_page_spans(const uint8_t *chunk, int64_t nbytes, int32_t codec, int32_t max_def_level, sb_page_span *out, int32_t cap,
                                     int32_t *out_n) {
  SB_API_BEGIN
  SB_REQUIRE(chunk && out && out_n && nbytes >= 0, "null argument");
  require_codec(codec);
  int32_t n = 0;
  walk_pages(chunk, nbytes, codec, max_def_level, false, cap, true, [&](const sb_page_span &sp) { out[n++] = sp; });
  *out_n = n;
  SB_API_END
}

static int phys_width_of(int32_t physical) {
  switch (physical) {
    case SB_PHYS_BOOLEAN: return 0;
    case SB_PHYS_INT32: case SB_PHYS_FLOAT: return 4;
    case SB_PHYS_INT64: case SB_PHYS_DOUBLE: return 8;
  }
  fail(SB_ERR_UNSUPPORTED, "Parquet physical type %d is not supported by the GPU scan (BOOLEAN, INT32, INT64, FLOAT, DOUBLE are)", physical);
}

// [offset, offset + bytes) lies inside a chunk of chunk_bytes bytes (written so that no sum can overflow)
static bool in_chunk(int64_t offset, int64_t bytes, int64_t chunk_bytes) {
  return offset >= 0 && bytes >= 0 && offset <= chunk_bytes && bytes <= chunk_bytes - offset;
}

// host state of one sb_scan_decode call that the stream reads asynchronously (freed by a host function behind the kernels)
struct ScanKeep {
  std::vector<PageTask> tasks, delta_tasks, str_pages, dba_pages;
  std::vector<ColTask> ctasks;
  std::vector<StrColTask> stasks;
  std::vector<StrOutTask> outs;
  std::vector<int32_t> dict_cols, str_cols, totals32;
  std::vector<int64_t> totals;
};

// steps (a)-(e) above for the string columns of one call; the one stream synchronisation of a call that decodes strings
static void decode_strings(ScanKeep &k, sb_table *t, int64_t nrows, cudaStream_t st) {
  const int ncols = (int)k.stasks.size(), nstr = (int)k.str_cols.size();
  Scratch d_cols((int64_t)ncols * sizeof(StrColTask), st), d_pages((int64_t)k.str_pages.size() * sizeof(PageTask), st),
      d_which((int64_t)k.dict_cols.size() * 4, st);
  SB_CUDA(cudaMemcpyAsync(d_cols.ptr, k.stasks.data(), (size_t)ncols * sizeof(StrColTask), cudaMemcpyHostToDevice, st));
  if (!k.str_pages.empty()) SB_CUDA(cudaMemcpyAsync(d_pages.ptr, k.str_pages.data(), k.str_pages.size() * sizeof(PageTask), cudaMemcpyHostToDevice, st));
  if (!k.dict_cols.empty()) SB_CUDA(cudaMemcpyAsync(d_which.ptr, k.dict_cols.data(), k.dict_cols.size() * 4, cudaMemcpyHostToDevice, st));
  {
    KernelTimer kt("scan_decode_strings", st);
    if (!k.dict_cols.empty()) {
      str_dict_kernel<<<(unsigned)k.dict_cols.size(), SCAN_THREADS, 0, st>>>(d_cols.as<StrColTask>(), d_which.as<int32_t>());
      SB_LAUNCH_CHECK();
    }
    if (!k.str_pages.empty()) {
      str_page_kernel<<<(unsigned)k.str_pages.size(), SCAN_THREADS, 0, st>>>(d_pages.as<PageTask>(), d_cols.as<StrColTask>());
      SB_LAUNCH_CHECK();
    }
  }
  // (c) offsets and arena sizes
  Scratch d_off((int64_t)nstr * (nrows + 1) * 8 + 16, st), d_tot((int64_t)nstr * 8 + 16, st);
  k.totals.assign(nstr, 0);
  if (nrows > 0) {
    for (int j = 0; j < nstr; j++)
      exclusive_scan_i32_to_i64(k.stasks[k.str_cols[j]].rlen, d_off.as<int64_t>() + (int64_t)j * (nrows + 1), nrows, d_tot.as<int64_t>() + j, st);
    SB_CUDA(cudaMemcpyAsync(k.totals.data(), d_tot.ptr, (size_t)nstr * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  k.outs.assign(ncols, StrOutTask{});
  k.totals32.assign(nstr, 0);
  for (int j = 0; j < nstr; j++) {
    const int ci = k.str_cols[j];
    if (k.totals[j] > 0x7fffffffll)
      fail(SB_ERR_UNSUPPORTED, "column chunk %d: the decoded strings take %lld bytes, more than the 2^31 - 1 an int32-offset string column holds", ci,
           (long long)k.totals[j]);
    Column &col = t->cols[ci];
    col.data = buffer_alloc(k.totals[j] + 16, st);
    col.string_bytes = k.totals[j];
    k.totals32[j] = (int32_t)k.totals[j];
    SB_CUDA(cudaMemcpyAsync((int32_t *)col.offsets->ptr + nrows, &k.totals32[j], 4, cudaMemcpyHostToDevice, st));
    StrOutTask &o = k.outs[ci];
    o.off = d_off.as<int64_t>() + (int64_t)j * (nrows + 1);
    o.out_off = (int32_t *)col.offsets->ptr;
    o.arena = (uint8_t *)col.data->ptr;
    o.nrows = nrows;
  }
  if (nrows == 0) return;
  // (d), (e) the bytes
  KernelTimer kt("scan_copy_strings", st);
  const int grid = grid_for(nrows, SCAN_THREADS, rt().num_sms * 16);
  for (int j = 0; j < nstr; j++) {
    const int ci = k.str_cols[j];
    str_copy_kernel<<<grid, SCAN_THREADS, 0, st>>>(k.stasks[ci], k.outs[ci]);
    SB_LAUNCH_CHECK();
  }
  if (!k.dba_pages.empty()) {
    Scratch d_dba((int64_t)k.dba_pages.size() * sizeof(PageTask), st), d_outs((int64_t)ncols * sizeof(StrOutTask), st);
    SB_CUDA(cudaMemcpyAsync(d_dba.ptr, k.dba_pages.data(), k.dba_pages.size() * sizeof(PageTask), cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(d_outs.ptr, k.outs.data(), (size_t)ncols * sizeof(StrOutTask), cudaMemcpyHostToDevice, st));
    str_prefix_kernel<<<(unsigned)k.dba_pages.size(), 32, 0, st>>>(d_dba.as<PageTask>(), d_cols.as<StrColTask>(), d_outs.as<StrOutTask>());
    SB_LAUNCH_CHECK();
  }
}

// Descriptors and launches of one decode call.  device_bytes(chunk, temps) returns where chunk's bytes (the offsets of its pages
// and dictionary) lie on the device; it is called once per chunk, in order, and may queue the chunk's copy and keep its buffer
// in temps.  Returns the table; the caller owns it.
template <class DeviceBytes>
static sb_table *scan_decode_chunks(const sb_column_chunk *chunks, int32_t ncols, cudaStream_t st, DeviceBytes device_bytes) {
  int64_t nrows = -1;
  // the descriptor arrays are copied to the device asynchronously: they live on the heap until the stream has consumed them
  // (cudaLaunchHostFunc below), so the call returns without a host synchronisation and the next row group's copy can be queued
  // on another stream while this one decodes
  using Keep = ScanKeep;
  std::unique_ptr<Keep> keep(new Keep());
  std::vector<PageTask> &tasks = keep->tasks;
  std::vector<ColTask> &ctasks = keep->ctasks;
  std::vector<StrColTask> &stasks = keep->stasks;
  ctasks.resize(ncols);
  stasks.resize(ncols);
  std::vector<std::unique_ptr<Scratch>> temps;
  auto scratch = [&](int64_t bytes) -> void * {
    Scratch *s = new Scratch(bytes, st);
    temps.emplace_back(s);
    return s->ptr;
  };
  sb_table *t = nullptr;
  try {
    for (int ci = 0; ci < ncols; ci++) {
      const sb_column_chunk &ch = chunks[ci];
      SB_REQUIRE(ch.data && ch.pages && ch.npages >= 0, "column chunk %d: null buffers", ci);
      const bool is_str = ch.physical_type == SB_PHYS_BYTE_ARRAY;
      const int pw = is_str ? 0 : phys_width_of(ch.physical_type);
      const int ow = type_width(ch.type);
      if (is_str) {
        SB_REQUIRE(ch.type == SB_STRING, "column chunk %d: physical type BYTE_ARRAY decodes to SB_STRING only (got column type %d)", ci, ch.type);
      } else {
        SB_REQUIRE(ow > 0, "column chunk %d: string columns are decoded from physical type BYTE_ARRAY only", ci);
        SB_REQUIRE(pw == 0 ? ch.type == SB_BOOL : (pw == 8 ? ow == 8 : (ow <= 4 || ch.type == SB_DECIMAL64)), "column chunk %d: physical type %d cannot feed column type %d", ci,
                   ch.physical_type, ch.type);
        SB_REQUIRE(ch.value_multiplier >= 0 && (ch.value_multiplier <= 1 || (ch.physical_type == SB_PHYS_INT64 && (ch.type == SB_TIMESTAMP || ch.type == SB_INT64))),
                   "column chunk %d: value multiplier %d applies to INT64 timestamp / long columns only", ci, ch.value_multiplier);
      }
      // an all-NULL chunk has an empty dictionary page; an entry takes at least 4 bytes (a PLAIN byte array's length) or its
      // physical width (one byte for BOOLEAN)
      const bool has_dict = ch.dict_offset >= 0 && ch.dict_count >= 0;
      SB_REQUIRE(!has_dict || in_chunk(ch.dict_offset, (int64_t)ch.dict_count * (is_str ? 4 : std::max(pw, 1)), ch.data_bytes),
                 "column chunk %d: dictionary overruns the chunk", ci);
      const uint8_t *dev = device_bytes(ch, temps);
      int64_t rows = 0;
      bool nullable = false, has_dba = false;
      for (int p = 0; p < ch.npages; p++) {
        const sb_page &pg = ch.pages[p];
        const int32_t e = pg.encoding;
        SB_REQUIRE(pg.num_values >= 0, "column chunk %d page %d has a negative value count (%d)", ci, p, pg.num_values);
        SB_REQUIRE(in_chunk(pg.values_offset, pg.values_bytes, ch.data_bytes) && in_chunk(pg.def_offset, pg.def_bytes, ch.data_bytes),
                   "column chunk %d page %d: offsets outside the chunk", ci, p);
        SB_REQUIRE(e == SB_ENC_PLAIN || (e == SB_ENC_RLE_DICTIONARY && has_dict) ||
                       (is_str ? e == SB_ENC_DELTA_LENGTH_BYTE_ARRAY || e == SB_ENC_DELTA_BYTE_ARRAY
                               : (e == SB_ENC_RLE_BOOLEAN && pw == 0) ||
                                     (e == SB_ENC_DELTA_BINARY_PACKED && (ch.physical_type == SB_PHYS_INT32 || ch.physical_type == SB_PHYS_INT64))),
                   "column chunk %d page %d: encoding %d%s", ci, p, e,
                   e == SB_ENC_RLE_DICTIONARY ? " without a dictionary page" : is_str ? " is not supported for BYTE_ARRAY columns" : " is not supported for this column");
        PageTask pt;
        pt.values = dev + pg.values_offset;
        pt.values_bytes = pg.values_bytes;
        pt.def = pg.def_bytes > 0 ? dev + pg.def_offset : nullptr;
        pt.def_bytes = pg.def_bytes;
        pt.row_start = rows;
        pt.num_values = pg.num_values;
        pt.encoding = e;
        pt.col = ci;
        pt.pad = 0;
        if (!is_str) {
          (e == SB_ENC_DELTA_BINARY_PACKED ? keep->delta_tasks : tasks).push_back(pt);
        } else if (pg.num_values > 0) {
          keep->str_pages.push_back(pt);
          if (e == SB_ENC_DELTA_BYTE_ARRAY) keep->dba_pages.push_back(pt);
        }
        rows += pg.num_values;
        nullable |= pg.def_bytes > 0;
        has_dba |= e == SB_ENC_DELTA_BYTE_ARRAY;
      }
      if (nrows < 0) {
        nrows = rows;
        t = table_new(nrows);
      }
      SB_REQUIRE(rows == nrows, "column chunk %d has %lld rows, chunk 0 has %lld", ci, (long long)rows, (long long)nrows);
      if (is_str) {
        Column col;
        col.type = SB_STRING;
        col.length = nrows;
        col.null_count = nullable ? -1 : 0;
        col.offsets = buffer_alloc((nrows + 1) * 4 + 16, st);
        if (nullable) col.validity = buffer_alloc(bitmap_alloc_bytes(nrows), st);
        t->cols.push_back(col);
        StrColTask &sc = stasks[ci];
        memset(&sc, 0, sizeof(sc));
        sc.base = dev;
        sc.data_bytes = ch.data_bytes;
        sc.rlen = (int32_t *)scratch(nrows * 4 + 16);
        sc.rsrc = (int64_t *)scratch(nrows * 8 + 16);
        sc.rpre = has_dba ? (int32_t *)scratch(nrows * 4 + 16) : nullptr;
        if (nullable) {
          sc.valid_bytes = (uint8_t *)scratch(nrows + 16);
          sc.vlen = (int32_t *)scratch(nrows * 4 + 16);
          sc.vsrc = (int64_t *)scratch(nrows * 8 + 16);
          sc.vpre = has_dba ? (int32_t *)scratch(nrows * 4 + 16) : nullptr;
        }
        ctasks[ci].valid_bytes = sc.valid_bytes;
        if (has_dict) {
          sc.dict_offset = ch.dict_offset;
          sc.dict_count = ch.dict_count;
          sc.dict_len = (int32_t *)scratch((int64_t)ch.dict_count * 4 + 16);
          sc.dict_src = (int64_t *)scratch((int64_t)ch.dict_count * 8 + 16);
          if (ch.dict_count > 0) keep->dict_cols.push_back(ci);
        }
        keep->str_cols.push_back(ci);
        continue;
      }
      Column col = column_alloc(ch.type, ch.scale, nrows, nullable, st);
      t->cols.push_back(col);
      ColTask &ct = ctasks[ci];
      ct.out = col.data->ptr;
      ct.valid_bytes = nullptr;
      ct.dense = nullptr;
      if (nullable) {
        Scratch *vb = new Scratch(nrows + 16, st), *dn = new Scratch(nrows * ow + 16, st);
        temps.emplace_back(vb);
        temps.emplace_back(dn);
        ct.valid_bytes = vb->as<uint8_t>();
        ct.dense = dn->as<uint8_t>();
      }
      ct.dict = has_dict ? dev + ch.dict_offset : nullptr;
      ct.dict_count = has_dict ? ch.dict_count : 0;
      ct.phys_width = pw;
      ct.out_width = ow;
      ct.mul = ch.value_multiplier;
    }
    std::vector<PageTask> &dtasks = keep->delta_tasks;
    const bool queued = nrows > 0 && (!tasks.empty() || !dtasks.empty());
    if (queued) {
      Scratch d_pages((int64_t)(tasks.size() + dtasks.size()) * sizeof(PageTask), st), d_cols((int64_t)ncols * sizeof(ColTask), st);
      if (!tasks.empty()) SB_CUDA(cudaMemcpyAsync(d_pages.ptr, tasks.data(), tasks.size() * sizeof(PageTask), cudaMemcpyHostToDevice, st));
      if (!dtasks.empty())
        SB_CUDA(cudaMemcpyAsync(d_pages.as<PageTask>() + tasks.size(), dtasks.data(), dtasks.size() * sizeof(PageTask), cudaMemcpyHostToDevice, st));
      SB_CUDA(cudaMemcpyAsync(d_cols.ptr, ctasks.data(), (size_t)ncols * sizeof(ColTask), cudaMemcpyHostToDevice, st));
      {
        KernelTimer kt("scan_decode", st);
        if (!tasks.empty()) {
          // enough blocks to fill the machine: pages of hybrid-encoded values are striped over `nparts` blocks each
          int nparts = (int)((rt().num_sms * 6 + (int64_t)tasks.size() - 1) / (int64_t)tasks.size());
          nparts = nparts < 1 ? 1 : (nparts > 16 ? 16 : nparts);
          scan_decode_kernel<<<(unsigned)(tasks.size() * nparts), SCAN_THREADS, 0, st>>>(d_pages.as<PageTask>(), d_cols.as<ColTask>(), nparts);
          SB_LAUNCH_CHECK();
        }
        if (!dtasks.empty()) {
          scan_delta_kernel<<<(unsigned)dtasks.size(), SCAN_THREADS, 0, st>>>(d_pages.as<PageTask>() + tasks.size(), d_cols.as<ColTask>());
          SB_LAUNCH_CHECK();
        }
      }
    }
    if (!keep->str_cols.empty()) decode_strings(*keep, t, nrows, st);
    if (queued || !keep->str_cols.empty()) {
      if (nrows > 0)
        for (int ci = 0; ci < ncols; ci++)
          if (ctasks[ci].valid_bytes) bytes_to_bitmap(ctasks[ci].valid_bytes, nrows, (uint32_t *)t->cols[ci].validity->ptr, st);
      Keep *raw = keep.release();
      if (cudaLaunchHostFunc(st, [](void *p) { delete (Keep *)p; }, raw) != cudaSuccess) {
        cudaGetLastError();
        cudaStreamSynchronize(st);
        delete raw;
      }
    }
  } catch (...) {
    if (t) table_free(t);
    throw;
  }
  return t;
}

extern "C" int sb_scan_decode(const sb_column_chunk *chunks, int32_t ncols, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(chunks && out && ncols > 0, "null argument");
  cudaStream_t st = stream_of(s);
  *out = scan_decode_chunks(chunks, ncols, st, [st](const sb_column_chunk &ch, std::vector<std::unique_ptr<Scratch>> &temps) {
    // the encoded bytes cross PCIe once, as they lie in the file
    Scratch *dev = new Scratch(ch.data_bytes + 32, st);
    temps.emplace_back(dev);
    if (ch.data_bytes > 0) SB_CUDA(cudaMemcpyAsync(dev->ptr, ch.data, (size_t)ch.data_bytes, cudaMemcpyHostToDevice, st));
    return (const uint8_t *)dev->ptr;
  });
  SB_API_END
}

// Compressed chunks: (1) one H2D copy per chunk; (2) scan_snappy decodes every page of the call into one image per chunk (page
// p at img_off[p], its size from the spans, so nothing is read back to allocate it); (3) scan_resolve_pages writes one record per
// page (status, V1 level length, first bytes of the values), read back with one synchronisation; (4) the host checks them as
// sb_parquet_chunk_pages checks the pages of a file, builds sb_page descriptors relative to the image and hands the images to
// scan_decode_chunks.
extern "C" int sb_scan_decode_compressed(const sb_compressed_chunk *chunks, int32_t ncols, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(chunks && out && ncols > 0, "null argument");
  cudaStream_t st = stream_of(s);
  std::vector<std::vector<int64_t>> img_off(ncols);
  std::vector<int64_t> img_bytes(ncols, 0);
  std::vector<std::unique_ptr<Scratch>> raw, images;
  std::vector<SnappyPage> sp;
  std::vector<ResolveTask> rt_tasks;
  std::vector<int32_t> slot_base(ncols, 0);
  for (int ci = 0; ci < ncols; ci++) {
    const sb_compressed_chunk &ch = chunks[ci];
    SB_REQUIRE(ch.data && (ch.spans || ch.npages == 0) && ch.npages >= 0 && ch.data_bytes >= 0, "column chunk %d: null buffers", ci);
    require_codec(ch.codec);
    SB_REQUIRE(ch.max_def_level == 0 || ch.max_def_level == 1, "column chunk %d: nested schemas are not supported (max definition level %d)", ci,
               ch.max_def_level);
    img_off[ci].resize(ch.npages);
    int64_t off = 0;
    for (int p = 0; p < ch.npages; p++) {
      const sb_page_span &x = ch.spans[p];
      SB_REQUIRE(in_chunk(x.body_offset, x.compressed_bytes, ch.data_bytes) && x.uncompressed_bytes >= 0 && x.levels_bytes >= 0 &&
                     x.levels_bytes <= x.compressed_bytes && x.levels_bytes <= x.uncompressed_bytes,
                 "column chunk %d page %d: span outside the chunk", ci, p);
      SB_REQUIRE(x.num_values >= 0, "column chunk %d page %d has a negative value count (%d)", ci, p, x.num_values);
      SB_REQUIRE(x.values_compressed ? ch.codec == SB_CODEC_SNAPPY : x.compressed_bytes == x.uncompressed_bytes,
                 "column chunk %d page %d: %s page of %d stored bytes for %d", ci, p, x.values_compressed ? "compressed" : "uncompressed",
                 x.compressed_bytes, x.uncompressed_bytes);
      img_off[ci][p] = off;
      off += ((int64_t)x.uncompressed_bytes + 15) / 16 * 16;
    }
    img_bytes[ci] = off;
    slot_base[ci] = (int32_t)sp.size();
    Scratch *r = new Scratch(ch.data_bytes + 16, st), *im = new Scratch(off + 32, st);
    raw.emplace_back(r);
    images.emplace_back(im);
    if (ch.data_bytes > 0) SB_CUDA(cudaMemcpyAsync(r->ptr, ch.data, (size_t)ch.data_bytes, cudaMemcpyHostToDevice, st));
    for (int p = 0; p < ch.npages; p++) {
      const sb_page_span &x = ch.spans[p];
      SnappyPage t;
      t.src = r->as<uint8_t>() + x.body_offset;
      t.dst = im->as<uint8_t>() + img_off[ci][p];
      t.levels_bytes = x.levels_bytes;
      t.src_bytes = x.compressed_bytes;
      t.dst_bytes = x.uncompressed_bytes;
      t.compressed = x.values_compressed != 0;
      t.slot = (int32_t)sp.size();
      sp.push_back(t);
      ResolveTask q;
      q.image = t.dst;
      q.bytes = x.uncompressed_bytes;
      q.levels_bytes = x.page_type == 3 ? x.levels_bytes : 0;
      q.v1_def = x.page_type == 0 && ch.max_def_level > 0;
      q.slot = t.slot;
      rt_tasks.push_back(q);
    }
  }
  const int np = (int)sp.size();
  std::vector<PageRecord> recs(np);
  if (np > 0) {
    // largest pages first: the block scheduler hands them out in order, so the longest page does not start last
    std::vector<SnappyPage> order(sp);
    std::stable_sort(order.begin(), order.end(), [](const SnappyPage &a, const SnappyPage &b) { return a.src_bytes > b.src_bytes; });
    Scratch d_sp((int64_t)np * sizeof(SnappyPage), st), d_rt((int64_t)np * sizeof(ResolveTask), st), d_status((int64_t)np * 4, st),
        d_rec((int64_t)np * sizeof(PageRecord), st);
    SB_CUDA(cudaMemcpyAsync(d_sp.ptr, order.data(), (size_t)np * sizeof(SnappyPage), cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(d_rt.ptr, rt_tasks.data(), (size_t)np * sizeof(ResolveTask), cudaMemcpyHostToDevice, st));
    {
      KernelTimer kt("scan_snappy", st);
      launch_snappy(d_sp.as<SnappyPage>(), np, d_status.as<int32_t>(), st);
    }
    {
      KernelTimer kt("scan_resolve_pages", st);
      launch_resolve_pages(d_rt.as<ResolveTask>(), np, d_status.as<int32_t>(), d_rec.as<PageRecord>(), st);
    }
    SB_CUDA(cudaMemcpyAsync(recs.data(), d_rec.ptr, (size_t)np * sizeof(PageRecord), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  raw.clear();
  // the descriptors sb_parquet_chunk_pages builds, over the decoded pages
  std::vector<ChunkPages> pages(ncols);
  std::vector<sb_column_chunk> dec(ncols);
  for (int ci = 0; ci < ncols; ci++) {
    const sb_compressed_chunk &ch = chunks[ci];
    for (int p = 0; p < ch.npages; p++) {
      const sb_page_span &x = ch.spans[p];
      const PageRecord &r = recs[slot_base[ci] + p];
      if (r.status != SNAPPY_OK)
        fail(SB_ERR_INVALID, "column chunk %d page %d (byte %lld of the column chunk): malformed Snappy stream: %s", ci, p,
             (long long)(x.body_offset - x.header_bytes), snappy_status_text(r.status));
      pages[ci].add(x, ch.max_def_level, img_off[ci][p], r.body_short ? nullptr : (const uint8_t *)&r.def_len, [&](const sb_page &pg) {
        return std::make_pair((const uint8_t *)r.head, std::min<int64_t>(r.head_bytes, pg.values_bytes));
      });
    }
    sb_column_chunk &d = dec[ci];
    memset(&d, 0, sizeof(d));
    d.type = ch.type;
    d.scale = ch.scale;
    d.physical_type = ch.physical_type;
    d.value_multiplier = ch.value_multiplier;
    d.data = images[ci]->as<uint8_t>();   // the image (device); scan_decode_chunks reads it through device_bytes only
    d.data_bytes = img_bytes[ci];
    d.pages = pages[ci].pages.data();
    d.npages = (int32_t)pages[ci].pages.size();
    d.dict_offset = pages[ci].dict_offset;
    d.dict_count = pages[ci].dict_count;
  }
  *out = scan_decode_chunks(dec.data(), ncols, st, [&](const sb_column_chunk &ch, std::vector<std::unique_ptr<Scratch>> &) { return ch.data; });
  SB_API_END
}

// Write-side twin for tests and bench.py: encodes one fixed-width column of `t` as a column chunk in the layout
// sb_scan_decode reads.  dictionary == nullptr: PLAIN pages.  Otherwise `dictionary` is a one-column table holding the
// column's distinct values in ascending order (e.g. sb_hash_aggregate with no aggregates + sb_sort; a float column's distinct
// bit patterns as integers, so -0.0 and each NaN payload are entries of their own): the chunk is
// [PLAIN dictionary values][pages of bit-packed indices].  The chunk stays on the device (out_chunk: one SB_INT8 column of
// bytes); page descriptors come back on the host.  No NULLs (definition levels are not written).
extern "C" int sb_scan_encode(const sb_table *t, int32_t col, const sb_table *dictionary, int64_t page_rows, sb_stream *s, sb_table **out_chunk,
                              sb_page *out_pages, int32_t pages_cap, int32_t *out_npages, int64_t *out_dict_offset, int32_t *out_dict_count) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(t && out_chunk && out_pages && out_npages && out_dict_offset && out_dict_count, "null argument");
  SB_REQUIRE(col >= 0 && col < (int)t->cols.size(), "column %d out of range", col);
  const Column &c = t->cols[col];
  SB_REQUIRE(c.type != SB_STRING && c.type != SB_BOOL && !c.validity, "sb_scan_encode takes NULL-free fixed-width numeric columns");
  const int ow = type_width(c.type), pw = ow == 8 ? 8 : 4;
  SB_REQUIRE(page_rows > 0 && page_rows % 8 == 0, "page_rows must be a positive multiple of 8");
  cudaStream_t st = stream_of(s);
  const int64_t n = t->nrows;
  const int64_t npages = n == 0 ? 0 : (n + page_rows - 1) / page_rows;
  SB_REQUIRE(npages <= pages_cap, "%lld pages do not fit the descriptor array (%d)", (long long)npages, pages_cap);
  sb_table *chunk = nullptr;
  if (!dictionary) {
    SB_REQUIRE(pw == ow, "PLAIN pages of %d-byte columns need a widening writer (dictionary-encode them)", ow);
    chunk = table_new(n * ow);
    Column bytes = column_alloc(SB_INT8, 0, n * ow, false, st);
    chunk->cols.push_back(bytes);
    if (n > 0) SB_CUDA(cudaMemcpyAsync(bytes.data->ptr, c.d(), (size_t)(n * ow), cudaMemcpyDeviceToDevice, st));
    for (int64_t p = 0; p < npages; p++) {
      sb_page &pg = out_pages[p];
      memset(&pg, 0, sizeof(pg));
      const int64_t lo = p * page_rows, hi = std::min(n, lo + page_rows);
      pg.encoding = SB_ENC_PLAIN;
      pg.num_values = (int32_t)(hi - lo);
      pg.values_offset = lo * ow;
      pg.values_bytes = (hi - lo) * ow;
    }
    *out_dict_offset = -1;
    *out_dict_count = 0;
  } else {
    // floats: the dictionary holds bit patterns (integers of the same width), searched in signed integer order
    const int32_t dict_type = c.type == SB_FLOAT32 ? SB_INT32 : c.type == SB_FLOAT64 ? SB_INT64 : c.type;
    SB_REQUIRE(dictionary->cols.size() == 1 && dictionary->cols[0].type == dict_type && !dictionary->cols[0].validity,
               "dictionary must be one NULL-free column of type %d (the column's type; the bit patterns of a float column)", dict_type);
    const int64_t dcount = dictionary->nrows;
    SB_REQUIRE(dcount >= 1 && dcount <= (1 << 24), "dictionary of %lld entries", (long long)dcount);
    int bw = 0;
    while ((1ll << bw) < dcount) bw++;
    if (bw == 0) bw = 1;   // keep one bit per value so every page has real runs
    const int64_t dict_bytes = (dcount * pw + 15) / 16 * 16;
    const int64_t full = page_rows / 504, tail = page_rows - full * 504;
    const int64_t page_stride = (1 + full * (1 + 63 * (int64_t)bw) + (tail ? 1 + ((tail + 7) / 8) * bw : 0) + 15) / 16 * 16;
    const int64_t total = dict_bytes + npages * page_stride;
    chunk = table_new(total);
    Column bytes = column_alloc(SB_INT8, 0, total, false, st);
    chunk->cols.push_back(bytes);
    uint8_t *base = (uint8_t *)bytes.data->ptr;
    SB_CUDA(cudaMemsetAsync(base, 0, (size_t)total, st));
    // dictionary page payload: PLAIN values at the physical width (INT32 for 1/2/4-byte columns)
    if (pw == ow) SB_CUDA(cudaMemcpyAsync(base, dictionary->cols[0].d(), (size_t)(dcount * ow), cudaMemcpyDeviceToDevice, st));
    else {
      std::vector<uint8_t> hv((size_t)(dcount * ow));
      SB_CUDA(cudaMemcpyAsync(hv.data(), dictionary->cols[0].d(), hv.size(), cudaMemcpyDeviceToHost, st));
      SB_CUDA(cudaStreamSynchronize(st));
      std::vector<int32_t> wide((size_t)dcount);
      for (int64_t i = 0; i < dcount; i++) wide[i] = ow == 1 ? (int32_t)((int8_t *)hv.data())[i] : (int32_t)((int16_t *)hv.data())[i];
      SB_CUDA(cudaMemcpyAsync(base, wide.data(), (size_t)dcount * 4, cudaMemcpyHostToDevice, st));
      SB_CUDA(cudaStreamSynchronize(st));
    }
    if (npages > 0) {
      uint8_t *pages_base = base + dict_bytes;
      const void *dv = dictionary->cols[0].d();
      switch (c.type) {
        case SB_INT8: encode_dict_pages_kernel<int8_t><<<(unsigned)npages, SCAN_THREADS, 0, st>>>((const int8_t *)c.d(), n, (const int8_t *)dv, (int32_t)dcount, bw, page_rows, page_stride, pages_base); break;
        case SB_INT16: encode_dict_pages_kernel<int16_t><<<(unsigned)npages, SCAN_THREADS, 0, st>>>((const int16_t *)c.d(), n, (const int16_t *)dv, (int32_t)dcount, bw, page_rows, page_stride, pages_base); break;
        case SB_INT32: case SB_DATE32: case SB_FLOAT32: encode_dict_pages_kernel<int32_t><<<(unsigned)npages, SCAN_THREADS, 0, st>>>((const int32_t *)c.d(), n, (const int32_t *)dv, (int32_t)dcount, bw, page_rows, page_stride, pages_base); break;
        default: encode_dict_pages_kernel<int64_t><<<(unsigned)npages, SCAN_THREADS, 0, st>>>((const int64_t *)c.d(), n, (const int64_t *)dv, (int32_t)dcount, bw, page_rows, page_stride, pages_base); break;
      }
      SB_LAUNCH_CHECK();
    }
    for (int64_t p = 0; p < npages; p++) {
      sb_page &pg = out_pages[p];
      memset(&pg, 0, sizeof(pg));
      const int64_t lo = p * page_rows, hi = std::min(n, lo + page_rows), rows = hi - lo;
      const int64_t fr = rows / 504, tl = rows - fr * 504;
      pg.encoding = SB_ENC_RLE_DICTIONARY;
      pg.num_values = (int32_t)rows;
      pg.values_offset = dict_bytes + p * page_stride;
      pg.values_bytes = 1 + fr * (1 + 63 * (int64_t)bw) + (tl ? 1 + ((tl + 7) / 8) * bw : 0);
    }
    *out_dict_offset = 0;
    *out_dict_count = (int32_t)dcount;
  }
  *out_npages = (int32_t)npages;
  *out_chunk = chunk;
  SB_API_END
}
