// snappy.cu -- raw Snappy blocks (the page bodies of parquet-mr / parquet-cpp SNAPPY chunks) decompressed on the GPU.
//
// Format (google/snappy format_description.txt): a varint preamble (the decompressed length, 1-5 bytes), then elements.  Tag
// byte & 3: 0 literal (length - 1 in the tag's upper 6 bits, or for 60..63 in 1..4 little-endian bytes after it, then the bytes),
// 1 copy with a 1-byte offset (length 4..11, 11-bit offset), 2 copy with a 2-byte offset, 3 copy with a 4-byte offset (length
// 1..64).  A copy appends out[p] = out[p - offset] byte by byte, so an overlapping copy (offset < length) repeats its first
// `offset` bytes: out[start + j] = out[start - offset + j mod offset].
//
// One 256-thread block per page, looping over windows of SN_WIN compressed bytes staged in shared memory:
//   parse    every byte of the window is a candidate element start; each thread computes the next element start of 16 of them
//            (speculatively: most candidates are not element starts).  The real chain from the window's first element is then
//            found by pointer jumping (mark the members reached so far, double the jumps) in log2(chain length) rounds, and the
//            members are compacted in order.  A block scan of their output lengths gives each element's output offset.
//   execute  consecutive copies with the same offset form one periodic run, so each output byte is a function of bytes that
//            are already final.  Wave 0 writes every literal and every copy whose source ends before the window's first output
//            byte; each following wave writes the copies whose sources end before the first copy not yet written.  In each
//            wave the active bytes are spread over all threads (flat index -> element by binary search).
// Every read is clamped to the page's compressed span and every write to its declared span; a malformed stream stops at its
// first bad element with a status (snappy.cuh), never reads or writes past its page.  The stream is accepted exactly when
// libsnappy would accept it and its preamble equals the page header's uncompressed size.
#include <climits>
#include "snappy.cuh"

namespace sb {

namespace {
constexpr int SN_THREADS = 256;
constexpr int SN_WIN = 4096;                   // compressed bytes parsed per window
constexpr int SN_PER = SN_WIN / SN_THREADS;    // candidate starts per thread
constexpr int SN_MAXE = SN_WIN / 2;            // every element takes at least 2 bytes
constexpr int SN_EPT = SN_MAXE / SN_THREADS;   // elements per thread
constexpr int SN_NW = SN_THREADS / 32;
constexpr uint16_t SN_SINK = SN_WIN;

struct SnSmem {
  uint8_t in[SN_WIN + 8];
  union {
    struct {
      uint16_t jump[SN_WIN + 2];
      uint8_t mark[SN_WIN + 4];
    } p;
    struct {
      uint32_t flat[SN_MAXE + 2];              // wave-active bytes before each element
      uint8_t lit[SN_MAXE];
    } x;
  } u;
  uint16_t epos[SN_MAXE];                      // element start in the window
  uint16_t head[SN_MAXE];                      // copy: first element of its run
  uint32_t eout[SN_MAXE + 1];                  // output offset from the window's first output byte
  uint32_t esrc[SN_MAXE];                      // literal: input position of its bytes; copy: offset
  int64_t w64[SN_NW];
  int32_t w32[SN_NW];
  int64_t in_pos, out_pos, next_in;
  int32_t status, err;
};

// element at window position i: header length (tag + extra bytes), output length, copy offset; false if the header does not
// fit in the window's wn bytes
__device__ __forceinline__ bool sn_element(const uint8_t *s, int i, int wn, int &hl, int64_t &len, uint32_t &off, bool &lit) {
  const uint32_t tag = s[i];
  off = 0;
  lit = (tag & 3) == 0;
  switch (tag & 3) {
    case 0: {
      const uint32_t l = tag >> 2;
      if (l < 60) {
        hl = 1;
        len = (int64_t)l + 1;
      } else {
        const int k = (int)l - 59;
        hl = 1 + k;
        uint32_t v = 0;
        for (int b = 0; b < k; b++) v |= (uint32_t)s[i + 1 + b] << (8 * b);   // s is padded: reads past wn are zeros
        len = (int64_t)v + 1;
      }
      break;
    }
    case 1:
      hl = 2;
      len = ((tag >> 2) & 7) + 4;
      off = ((tag >> 5) << 8) | s[i + 1];
      break;
    case 2:
      hl = 3;
      len = (tag >> 2) + 1;
      off = (uint32_t)s[i + 1] | ((uint32_t)s[i + 2] << 8);
      break;
    default:
      hl = 5;
      len = (tag >> 2) + 1;
      off = (uint32_t)s[i + 1] | ((uint32_t)s[i + 2] << 8) | ((uint32_t)s[i + 3] << 16) | ((uint32_t)s[i + 4] << 24);
      break;
  }
  return i + hl <= wn;
}

// exclusive block scan; *total = op over the block.  All threads call it.
template <class T, class Op>
__device__ __forceinline__ T sn_scan(T x, T identity, Op op, T *wbuf, T *total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  T incl = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl = op(incl, o);
  }
  if (lane == 31) wbuf[w] = incl;
  __syncthreads();
  T base = identity, tot = identity;
#pragma unroll
  for (int k = 0; k < SN_NW; k++) {
    if (k < w) base = op(base, wbuf[k]);
    tot = op(tot, wbuf[k]);
  }
  __syncthreads();
  T ex = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) ex = identity;
  *total = tot;
  return op(base, ex);
}
struct SnAdd {
  __device__ int64_t operator()(int64_t a, int64_t b) const { return a + b; }
};
struct SnMax {
  __device__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};
struct SnMin {
  __device__ int64_t operator()(int64_t a, int64_t b) const { return a < b ? a : b; }
};

__device__ void snappy_block(const uint8_t *__restrict__ in, int64_t nin, uint8_t *__restrict__ out, int64_t nout, SnSmem &sm) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    uint32_t v = 0;
    int l = 0, st = SNAPPY_OK;
    while (true) {
      if (l >= nin) { st = SNAPPY_BAD_PREAMBLE; break; }
      const uint32_t b = in[l];
      if (l == 4 && b >= 16) { st = SNAPPY_BAD_PREAMBLE; break; }   // more than 32 bits, or a sixth byte
      v |= (b & 0x7f) << (7 * l);
      l++;
      if (!(b & 0x80)) break;
    }
    if (st == SNAPPY_OK && (int64_t)v != nout) st = SNAPPY_LENGTH_MISMATCH;
    sm.status = st;
    sm.in_pos = l;
    sm.out_pos = 0;
  }
  __syncthreads();
  while (true) {
    const int64_t w0 = sm.in_pos, ob = sm.out_pos;
    const int status = sm.status;
    __syncthreads();
    if (status != SNAPPY_OK) break;
    if (w0 >= nin) {
      if (tid == 0 && ob < nout) sm.status = SNAPPY_SHORT;
      break;
    }
    const int wn = (int)(nin - w0 < SN_WIN ? nin - w0 : SN_WIN);
    const bool at_end = w0 + wn >= nin;
    for (int i = tid; i < SN_WIN + 8; i += SN_THREADS) sm.in[i] = i < wn ? in[w0 + i] : 0;
    if (tid == 0) {
      sm.u.p.jump[SN_SINK] = SN_SINK;
      sm.u.p.mark[SN_SINK] = 0;
      sm.err = INT_MAX;
    }
    __syncthreads();
    // ---- parse: next element start of every candidate, then the chain from position 0 by pointer jumping ----------------
#pragma unroll 4
    for (int k = 0; k < SN_PER; k++) {
      const int i = tid * SN_PER + k;
      uint16_t j = SN_SINK;
      if (i < wn) {
        int hl;
        int64_t len;
        uint32_t off;
        bool lit;
        if (sn_element(sm.in, i, wn, hl, len, off, lit)) {
          const int64_t nx = i + hl + (lit ? len : 0);
          if (nx < wn) j = (uint16_t)nx;
        }
      }
      sm.u.p.jump[i] = j;
      sm.u.p.mark[i] = i == 0;
    }
    __syncthreads();
    while (true) {
      int grew = 0;
      for (int k = 0; k < SN_PER; k++) {
        const int i = tid * SN_PER + k;
        if (sm.u.p.mark[i]) {
          const int j = sm.u.p.jump[i];
          if (j != SN_SINK && !sm.u.p.mark[j]) {
            sm.u.p.mark[j] = 1;
            grew = 1;
          }
        }
      }
      if (!__syncthreads_or(grew)) break;
      uint16_t nj[SN_PER];
#pragma unroll
      for (int k = 0; k < SN_PER; k++) nj[k] = sm.u.p.jump[sm.u.p.jump[tid * SN_PER + k]];
      __syncthreads();
#pragma unroll
      for (int k = 0; k < SN_PER; k++) sm.u.p.jump[tid * SN_PER + k] = nj[k];
      __syncthreads();
    }
    int cnt = 0;
    for (int k = 0; k < SN_PER; k++) cnt += sm.u.p.mark[tid * SN_PER + k];
    int64_t nel64;
    int64_t at = sn_scan<int64_t>(cnt, 0, SnAdd(), sm.w64, &nel64);
    for (int k = 0; k < SN_PER; k++)
      if (sm.u.p.mark[tid * SN_PER + k]) sm.epos[at++] = (uint16_t)(tid * SN_PER + k);
    const int nel = (int)nel64;
    __syncthreads();
    // ---- elements: kind, source, output length; the errors of the earliest bad element win ----------------------------
    uint32_t olen[SN_EPT];
    uint8_t bad1[SN_EPT];
    int64_t mine = 0;
#pragma unroll
    for (int k = 0; k < SN_EPT; k++) {
      const int e = tid * SN_EPT + k;
      olen[k] = 0;
      bad1[k] = 0;
      if (e >= nel) continue;
      const int i = sm.epos[e];
      int hl;
      int64_t len;
      uint32_t off;
      bool lit;
      const bool whole = sn_element(sm.in, i, wn, hl, len, off, lit);
      int bad = 0;
      int64_t nx = i + hl + (lit ? len : 0);
      if (!whole) {                             // header cut by the window: the next window starts at it
        if (at_end) bad = SNAPPY_INPUT_OVERRUN;
        nx = i;
        len = 0;
        lit = true;
      } else if (lit && w0 + nx > nin) {
        bad = SNAPPY_INPUT_OVERRUN;
      } else if (!lit && off == 0) {
        bad = SNAPPY_BAD_OFFSET;
      }
      if (!bad && len > nout) bad = SNAPPY_OUTPUT_OVERRUN;
      bad1[k] = (uint8_t)bad;
      if (nx >= wn || !whole) sm.next_in = w0 + nx;   // the chain's last member
      sm.u.x.lit[e] = lit;
      sm.esrc[e] = lit ? (uint32_t)(w0 + i + hl) : off;
      olen[k] = bad ? 0 : (uint32_t)len;   // bad: the call fails before any byte is written
      mine += olen[k];
    }
    int64_t wtot;
    int64_t eo = sn_scan<int64_t>(mine, 0, SnAdd(), sm.w64, &wtot);
    int32_t hmax = -1;
#pragma unroll
    for (int k = 0; k < SN_EPT; k++) {
      const int e = tid * SN_EPT + k;
      if (e >= nel) continue;
      // an element that starts at or after the declared end is left over, whatever it is; else its own first fault
      int bad = ob + eo >= nout && (olen[k] > 0 || bad1[k]) ? SNAPPY_LEFTOVER : bad1[k];
      if (!bad && ob + eo + olen[k] > nout) bad = SNAPPY_OUTPUT_OVERRUN;
      if (!bad && !sm.u.x.lit[e] && ob + eo < (int64_t)sm.esrc[e]) bad = SNAPPY_BAD_OFFSET;
      if (bad) atomicMin(&sm.err, e * 16 + bad);
      sm.eout[e] = (uint32_t)eo;
      eo += olen[k];
      if (!sm.u.x.lit[e] && (e == 0 || sm.u.x.lit[e - 1] || sm.esrc[e - 1] != sm.esrc[e])) hmax = e;
    }
    int32_t hdummy;
    int32_t hbase = sn_scan<int32_t>(hmax, -1, SnMax(), sm.w32, &hdummy);
    if (sm.err != INT_MAX) {                     // written before the scan's barriers
      if (tid == 0) sm.status = sm.err & 15;
      __syncthreads();
      break;
    }
    // send[k]: output offset (from ob) where the bytes copy k reads end; a copy runs once every byte before that is final
    int64_t send[SN_EPT];
#pragma unroll
    for (int k = 0; k < SN_EPT; k++) {
      const int e = tid * SN_EPT + k;
      send[k] = 0;
      if (e >= nel || sm.u.x.lit[e]) continue;
      const bool is_head = e == 0 || sm.u.x.lit[e - 1] || sm.esrc[e - 1] != sm.esrc[e];
      if (is_head) hbase = e;
      sm.head[e] = (uint16_t)hbase;
      const int64_t oh = sm.eout[hbase], off = sm.esrc[e];
      const int64_t span = (int64_t)sm.eout[e] + olen[k] - oh;
      send[k] = oh - off + (span < off ? span : off);
    }
    if (tid == 0) sm.eout[nel] = (uint32_t)wtot;
    // ---- execute in waves ---------------------------------------------------------------------------------------------
    int64_t fprev = INT64_MIN, f = 0;
    for (int wave = 0;; wave++) {
      int64_t act = 0;
      uint32_t a[SN_EPT];
#pragma unroll
      for (int k = 0; k < SN_EPT; k++) {
        const int e = tid * SN_EPT + k;
        a[k] = 0;
        if (e >= nel) continue;
        const bool run = sm.u.x.lit[e] ? wave == 0 : (send[k] <= f && send[k] > fprev);
        a[k] = run ? olen[k] : 0;
        act += a[k];
      }
      int64_t total;
      int64_t fb = sn_scan<int64_t>(act, 0, SnAdd(), sm.w64, &total);
#pragma unroll
      for (int k = 0; k < SN_EPT; k++) {
        const int e = tid * SN_EPT + k;
        if (e < nel) sm.u.x.flat[e] = (uint32_t)fb;
        fb += a[k];
      }
      if (tid == 0) sm.u.x.flat[nel] = (uint32_t)total;
      __syncthreads();
      for (int64_t g0 = (int64_t)tid * 4; g0 < total; g0 += SN_THREADS * 4) {
        int lo = 0, hi = nel;                     // last element with flat <= g0 (it has active bytes)
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (sm.u.x.flat[mid] <= g0) lo = mid; else hi = mid;
        }
        int e = lo;
        for (int g = 0; g < 4; g++) {
          const int64_t fi = g0 + g;
          if (fi >= total) break;
          while (sm.u.x.flat[e + 1] <= fi) e++;
          const int64_t rel = (int64_t)sm.eout[e] + (fi - sm.u.x.flat[e]);
          uint8_t v;
          if (sm.u.x.lit[e]) {
            v = in[sm.esrc[e] + (rel - sm.eout[e])];
          } else {
            const uint32_t off = sm.esrc[e];
            const int64_t oh = ob + sm.eout[sm.head[e]];
            v = out[oh - off + (uint32_t)(ob + rel - oh) % off];
          }
          out[ob + rel] = v;
        }
      }
      __syncthreads();                            // this wave's bytes are final for the next one
      int64_t m = INT64_MAX;
#pragma unroll
      for (int k = 0; k < SN_EPT; k++) {
        const int e = tid * SN_EPT + k;
        if (e < nel && !sm.u.x.lit[e] && olen[k] > 0 && send[k] > f && (int64_t)sm.eout[e] < m) m = sm.eout[e];
      }
      int64_t fnext;
      sn_scan<int64_t>(m, INT64_MAX, SnMin(), sm.w64, &fnext);
      if (fnext == INT64_MAX) break;
      fprev = f;
      f = fnext;
    }
    if (tid == 0) {
      sm.in_pos = sm.next_in;
      sm.out_pos = ob + wtot;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(SN_THREADS) scan_snappy(const SnappyPage *__restrict__ pages, int32_t *__restrict__ status) {
  __shared__ SnSmem sm;
  const SnappyPage pg = pages[blockIdx.x];
  const int64_t copy = pg.compressed ? pg.levels_bytes : pg.src_bytes;   // level bytes, or the whole uncompressed body
  for (int64_t i = threadIdx.x; i < copy; i += SN_THREADS) pg.dst[i] = pg.src[i];
  if (!pg.compressed) {
    if (threadIdx.x == 0) status[pg.slot] = SNAPPY_OK;
    return;
  }
  snappy_block(pg.src + pg.levels_bytes, pg.src_bytes - pg.levels_bytes, pg.dst + pg.levels_bytes, pg.dst_bytes - pg.levels_bytes, sm);
  if (threadIdx.x == 0) status[pg.slot] = sm.status;
}

__global__ void scan_resolve_pages(const ResolveTask *__restrict__ tasks, int n, const int32_t *__restrict__ status, PageRecord *__restrict__ records) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ResolveTask t = tasks[i];
  PageRecord &r = records[t.slot];
  const int32_t st = status[t.slot];
  uint32_t def_len = 0;
  int32_t body_short = 0, head_bytes = 0;
  if (st == SNAPPY_OK) {
    int64_t vpos = t.levels_bytes;
    if (t.v1_def) {
      if (t.bytes < 4) {
        body_short = 1;
        vpos = t.bytes;
      } else {
        def_len = (uint32_t)t.image[0] | ((uint32_t)t.image[1] << 8) | ((uint32_t)t.image[2] << 16) | ((uint32_t)t.image[3] << 24);
        vpos = 4 + (int64_t)def_len;
      }
    }
    if (vpos < t.bytes) head_bytes = (int32_t)(t.bytes - vpos < PAGE_HEAD_BYTES ? t.bytes - vpos : PAGE_HEAD_BYTES);
    for (int b = 0; b < head_bytes; b++) r.head[b] = t.image[vpos + b];
  }
  for (int b = head_bytes; b < PAGE_HEAD_BYTES; b++) r.head[b] = 0;
  r.status = st;
  r.def_len = def_len;
  r.body_short = body_short;
  r.head_bytes = head_bytes;
}
}  // namespace

const char *snappy_status_text(int status) {
  switch (status) {
    case SNAPPY_BAD_PREAMBLE: return "truncated or overlong length preamble";
    case SNAPPY_LENGTH_MISMATCH: return "length preamble differs from the page header's uncompressed size";
    case SNAPPY_INPUT_OVERRUN: return "literal or tag past the end of the input";
    case SNAPPY_BAD_OFFSET: return "copy offset 0 or reaching before the page start";
    case SNAPPY_OUTPUT_OVERRUN: return "output past the declared length";
    case SNAPPY_LEFTOVER: return "bytes left over after the declared length";
    case SNAPPY_SHORT: return "stream ends before the declared length";
  }
  return "ok";
}

void launch_snappy(const SnappyPage *d_pages, int npages, int32_t *d_status, cudaStream_t st) {
  if (npages <= 0) return;
  scan_snappy<<<(unsigned)npages, SN_THREADS, 0, st>>>(d_pages, d_status);
  SB_LAUNCH_CHECK();
}

void launch_resolve_pages(const ResolveTask *d_tasks, int ntasks, const int32_t *d_status, PageRecord *d_records, cudaStream_t st) {
  if (ntasks <= 0) return;
  scan_resolve_pages<<<(unsigned)((ntasks + 127) / 128), 128, 0, st>>>(d_tasks, ntasks, d_status, d_records);
  SB_LAUNCH_CHECK();
}

}  // namespace sb
